"""One replica of a DiLoCo replica group on ``Manager`` + ``ProcessGroupB200``, recording every outer sync, for
``tests/test_diloco_exact_gpu.py``. Start one process per replica (``--replica 0``, ``1``, ``2``; they may share one
GPU); each runs the cases of ``--cases`` (a JSON list) in order, against the lighthouse address each case carries,
and skips the cases with fewer replicas than its index.

Wrappers around ``prepare_sync``, ``perform_sync`` and ``_perform_sync_flat`` observe and change nothing. Per sync they
write ``<out>/<case>/r<replica>_<k>.pt``:

* at prepare time, on the main stream: the fragment, the committed step, the process-group rank and size,
  ``num_participants()``, ``is_participating()``, and copies of ``flat_param`` and ``flat_orig``;
* around the fused kernel: the averaged ``flat_grad`` and ``flat_orig``, ``flat_param``, ``flat_mom`` before and after;
* the commit verdict and the whole parameter storage before and after the sync.

A case is a dict: ``name``, ``lighthouse``, ``replicas``, ``model`` (``llama``: llama3_tiny on ``FlatParams``;
``packed``: weights packed into one buffer, 16-byte aligned; ``packed_gap``: the same, with a small weight of fragment
1 between two weights of fragment 0 and the other way round; ``packed_tail``: packed with no padding, so fragment 0
ends off a multiple of 8), ``dtype``, ``quantize``, ``fragments``, ``delay``, ``alpha``, ``mu``, ``nesterov``, ``syncs`` (committed
outer steps to run), and optionally:

* ``spares``: ``WorldSizeMode.FIXED_WITH_SPARES`` with two contributors, so the third replica adds zeros;
* ``fail_at``: every replica calls ``manager.report_error`` before ``should_commit`` at that committed step (a
  host-side veto): every replica discards the sync and retries the fragment;
* ``join_after``: replica 2 starts once the others have committed that many outer steps, and heals;
* ``slow``: ``torch.cuda._sleep`` on the fragment's side stream ahead of the pseudo-gradient launch;
* ``mutant``: a deliberate Python-level defect (see ``MUTANTS``) the checks must catch.
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time
from datetime import timedelta
from typing import Any, Callable, Dict, List, Tuple

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WINDOW = 3  # inner steps per fragment window
SLEEP_CYCLES = 200_000_000  # ~0.1 s of side-stream delay: longer than an inner step of the tiny models
DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}


class _Frag(nn.Module):
    def __init__(self, params: List[nn.Parameter]) -> None:
        super().__init__()
        self.ps = nn.ParameterList(params)


def _packed(dev: torch.device, dtype: torch.dtype, sizes: List[int], align: int) -> Tuple[nn.Module, List[nn.Parameter]]:
    offs, total = [], 0
    for n in sizes:
        offs.append(total)
        total += (n + align - 1) // align * align
    buf = torch.zeros(total, dtype=dtype, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    params = []
    for o, n in zip(offs, sizes):
        buf[o:o + n] = torch.randn(n, device=dev, generator=gen).to(dtype)
        params.append(nn.Parameter(buf[o:o + n]))
    return _Frag(params), params


def build(case: Dict[str, Any], dev: torch.device) -> Tuple[nn.Module, List[List[nn.Parameter]], Any]:
    """The model, its fragments (lists of parameters) and how an inner step gets its gradients:
    ``("llama", (vocab_size, flat_params))`` runs the forward and backward on random tokens, ``("synthetic", None)``
    draws them."""
    kind = case["model"]
    if kind.startswith("llama"):
        from torchft_b200.models.llama import CONFIGS, FlatParams, Llama

        torch.manual_seed(0)
        cfg = CONFIGS["llama3_tiny"]
        model = Llama(cfg, device=dev)
        flat = FlatParams(model)
        model.init_weights(3)
        order = sorted(model.parameters(), key=lambda p: p.data_ptr())  # FlatParams order
        if case["fragments"] == 1:
            frags = [order]
        else:
            frags = [order[: len(order) // 2], order[len(order) // 2:]]
        return model, frags, ("llama", (cfg.vocab_size, flat))
    dtype = DTYPES[case["dtype"]]
    if kind == "packed_tail":
        model, ps = _packed(dev, dtype, [512, 500, 1000], 1)
        return model, [ps[:2], ps[2:]], ("synthetic", None)
    model, ps = _packed(dev, dtype, [1000, 24, 3000, 8, 520], 8)
    if kind == "packed_gap":  # each fragment's span holds a weight of the other within 4096 elements
        frags = [[ps[0], ps[2]], [ps[1], ps[3], ps[4]]]
    else:
        frags = [ps] if case["fragments"] == 1 else [ps[:2], ps[2:]]
    return model, frags, ("synthetic", None)


# ------------------------------------------------------------------------------------------------ mutants
def _mutant_alpha(patch: Callable[..., None]) -> None:
    from torchft_b200.ops import _native

    real = _native.load

    class Flip:
        def __init__(self, k: Any) -> None:
            self._k = k

        def __getattr__(self, name: str) -> Any:
            return getattr(self._k, name)

        def diloco_outer(self, *a: Any) -> Any:
            a = list(a)
            a[9] = 1.0 - a[9]
            return self._k.diloco_outer(*a)

    patch(_native, "load", lambda: Flip(real()))


def _mutant_heal_without_momentum(patch: Callable[..., None]) -> None:
    from torchft_b200.manager import Manager

    real = Manager.register_state_dict_fn

    def register(self: Any, key: str, load: Any, save: Any) -> None:
        def save_dropped() -> Any:
            sd = save()
            sd.pop("outer_momentum", None)
            return sd

        real(self, key, load, save_dropped if key.startswith("StreamingDiLoCoFragment") else save)

    patch(Manager, "register_state_dict_fn", register)


def _mutant_world_scale(patch: Callable[..., None]) -> None:
    from torchft_b200.manager import Manager

    patch(Manager, "num_participants", lambda self: self._pg.size())


def _mutant_race(patch: Callable[..., None]) -> None:
    from torchft_b200.local_sgd import _StreamingDiLoCoFragment

    patch(_StreamingDiLoCoFragment, "fence_weight_writes", lambda self: None)


def _mutant_span(patch: Callable[..., None]) -> None:
    from torchft_b200.local_sgd import _StreamingDiLoCoFragment

    patch(_StreamingDiLoCoFragment, "_span_is_own", lambda self, lo, hi: True)


MUTANTS = {
    "alpha": _mutant_alpha,  # diloco_outer merges with 1 - alpha
    "heal_without_momentum": _mutant_heal_without_momentum,  # outer_momentum left out of the heal state
    "world_scale": _mutant_world_scale,  # the average divides by the group size, not by the contributors
    "race": _mutant_race,  # the inner step does not wait for the pseudo-gradient's reads
    "span": _mutant_span,  # the flat span may cover weights of another fragment
}


# ------------------------------------------------------------------------------------------------ one case
def _wait_for(path: str, timeout: float = 240.0) -> None:
    deadline = time.monotonic() + timeout
    while not os.path.exists(path):
        if time.monotonic() > deadline:
            raise TimeoutError(f"{path} did not appear")
        time.sleep(0.05)


def run_case(case: Dict[str, Any], replica: int, out: str) -> None:
    from torchft_b200.local_sgd import DiLoCo, _StreamingDiLoCoFragment
    from torchft_b200.manager import Manager, WorldSizeMode
    from torchft_b200.parallel.process_group_b200 import ProcessGroupB200

    cdir = os.path.join(out, case["name"])
    os.makedirs(cdir, exist_ok=True)
    joiner = case.get("join_after") is not None and replica == 2
    if joiner:  # start once the others have committed join_after outer steps
        _wait_for(os.path.join(cdir, "joinable"))

    undo: List[Tuple[Any, str, Any]] = []

    def patch(obj: Any, name: str, value: Any) -> None:
        undo.append((obj, name, obj.__dict__.get(name, AttributeError)))
        setattr(obj, name, value)

    if case.get("mutant"):
        MUTANTS[case["mutant"]](patch)

    dev = torch.device("cuda", 0)
    model, frag_params, (kind, aux) = build(case, dev)
    params = [p for f in frag_params for p in f]
    es = params[0].element_size()
    store_t = torch.empty(0, dtype=params[0].dtype, device=dev).set_(
        params[0].untyped_storage(), 0, (params[0].untyped_storage().nbytes() // es,))
    base = store_t.data_ptr()
    table = [((p.data_ptr() - base) // es, p.numel(), fi) for fi, f in enumerate(frag_params) for p in f]

    store = torch.distributed.TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)
    pg = ProcessGroupB200(timeout=timedelta(seconds=30), device=dev)
    mode = WorldSizeMode.FIXED_WITH_SPARES if case.get("spares") else WorldSizeMode.DYNAMIC
    manager = Manager(pg=pg, min_replica_size=2, use_async_quorum=False, world_size_mode=mode,
                      load_state_dict=lambda sd: model.load_state_dict(sd), state_dict=lambda: model.state_dict(),
                      replica_id=f"{case['name']}_{replica}", store_addr="127.0.0.1", store_port=store.port, rank=0,
                      world_size=1, lighthouse_addr=case["lighthouse"], timeout=timedelta(seconds=30),
                      quorum_timeout=timedelta(seconds=60), connect_timeout=timedelta(seconds=30))

    records: List[Dict[str, Any]] = []
    pending: Dict[int, Dict[str, Any]] = {}
    vetoed: List[bool] = []

    def clone(t: Any) -> Any:
        return None if t is None else t.detach().clone()

    real_prepare = _StreamingDiLoCoFragment.prepare_sync
    real_perform = _StreamingDiLoCoFragment.perform_sync
    real_flat = _StreamingDiLoCoFragment._perform_sync_flat
    real_launch = _StreamingDiLoCoFragment._launch_pseudograd_allreduce

    def prepare_sync(self: Any) -> None:
        pending[self._fragment_id] = {
            "fragment": self._fragment_id, "step": manager.current_step(), "pg_rank": pg.rank(), "pg_world": pg.size(),
            "participants": manager._participation.world, "participating": manager.is_participating(),
            "snap_param": clone(self._flat_param), "snap_orig": clone(self._flat_orig)}
        real_prepare(self)

    def perform_sync(self: Any) -> bool:
        rec = pending[self._fragment_id]
        rec["storage_before"] = store_t.clone()
        if case.get("fail_at") == manager.current_step() and not vetoed:
            vetoed.append(True)
            manager.report_error(RuntimeError("injected veto"))
        rec["verdict"] = real_perform(self)
        print(f"[replica {replica}] {case['name']}: sync {len(records)} step {rec['step']} fragment {rec['fragment']} "
              f"commit {rec['verdict']}", flush=True)
        rec["storage_after"] = store_t.clone()
        torch.cuda.synchronize()
        records.append(pending.pop(self._fragment_id))
        return rec["verdict"]

    def perform_sync_flat(self: Any) -> bool:
        rec = pending[self._fragment_id]
        rec.update(grad=clone(self._flat_grad), orig_before=clone(self._flat_orig), param_before=clone(self._flat_param),
                   mom_before=clone(self._flat_mom))
        verdict = real_flat(self)
        rec.update(orig_after=clone(self._flat_orig), param_after=clone(self._flat_param), mom_after=clone(self._flat_mom))
        return verdict

    def launch(self: Any) -> None:
        torch.cuda._sleep(SLEEP_CYCLES)  # on the side stream: the pseudo-gradient starts late
        real_launch(self)

    patch(_StreamingDiLoCoFragment, "prepare_sync", prepare_sync)
    patch(_StreamingDiLoCoFragment, "perform_sync", perform_sync)
    patch(_StreamingDiLoCoFragment, "_perform_sync_flat", perform_sync_flat)
    if case.get("slow"):
        patch(_StreamingDiLoCoFragment, "_launch_pseudograd_allreduce", launch)

    n_frag = len(frag_params)
    frags = [_Frag(f) for f in frag_params]
    inner = torch.optim.SGD(params, lr=0.05)
    outers = [torch.optim.SGD(f.parameters(), lr=0.7, momentum=case["mu"], nesterov=case["nesterov"]) for f in frags]
    gen = torch.Generator(device=dev).manual_seed(100 + replica)
    try:
        with DiLoCo(manager, frags, inner, outers, sync_every=WINDOW * n_frag, backup_device=dev,
                    should_quantize=case["quantize"], fragment_sync_delay=case["delay"],
                    fragment_update_alpha=case["alpha"]) as d:
            flat = [f._flat_grad is not None for f in d._fragments]
            if case["model"] in ("llama", "packed"):
                assert all(flat), f"{case['name']}: the flat path was not taken: {flat}"
            if joiner:
                open(os.path.join(cdir, "ready"), "w").close()
            told = joiner or case.get("join_after") is None
            while manager.current_step() < case["syncs"]:
                if not told and manager.current_step() >= case["join_after"]:
                    # the others wait here, at a window boundary, until the late replica can ask for a quorum
                    if replica == 0:
                        open(os.path.join(cdir, "joinable"), "w").close()
                    _wait_for(os.path.join(cdir, "ready"))
                    told = True
                if kind == "llama":
                    # zeroed gradient views: the fused nodes write some gradients straight into the flat buffer, and a
                    # parameter whose .grad is None would be skipped by the inner optimizer
                    aux[1].reset_grads(zero=True)
                    tok = torch.randint(0, aux[0], (2, 32), device=dev, generator=gen)
                    tgt = torch.randint(0, aux[0], (2, 32), device=dev, generator=gen)
                    model(tok, tgt).backward()
                else:
                    for p in params:
                        p.grad = torch.randn(p.shape, device=dev, generator=gen).to(p.dtype)
                inner.step()
        torch.cuda.synchronize()
        meta = {"table": table, "flat": flat, "dtype": str(params[0].dtype), "syncs": len(records),
                "spans": [((f._flat_param.data_ptr() - base) // es, f._flat_param.numel()) if f._flat_param is not None
                          else None for f in d._fragments]}
        for k, rec in enumerate(records):
            torch.save({n: (v.cpu() if isinstance(v, torch.Tensor) else v) for n, v in rec.items()},
                       os.path.join(cdir, f"r{replica}_{k}.pt"))
        with open(os.path.join(cdir, f"r{replica}.json"), "w") as f:
            json.dump(meta, f)
    finally:
        for obj, name, old in reversed(undo):
            if old is AttributeError:
                delattr(obj, name)
            else:
                setattr(obj, name, old)
        manager.shutdown(wait=False)
        pg.shutdown()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--replica", type=int, required=True)
    ap.add_argument("--cases", required=True, help="JSON file: a list of case dicts")
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    with open(a.cases) as f:
        cases = json.load(f)
    failed = []
    for case in cases:
        if a.replica >= case["replicas"]:
            continue
        print(f"[replica {a.replica}] {case['name']}: start", flush=True)
        try:
            run_case(case, a.replica, a.out)
            print(f"[replica {a.replica}] {case['name']}: done", flush=True)
        except Exception as e:  # noqa: BLE001 - the others still run; the test reports the missing records
            import traceback

            traceback.print_exc()
            failed.append(f"{case['name']}: {e!r}")
    print(json.dumps({"replica": a.replica, "failed": failed}), flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
