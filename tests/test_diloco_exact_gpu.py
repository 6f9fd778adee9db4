"""The flat DiLoCo sync across 2 and 3 replica processes on one GPU, held sync by sync to an exact replay of the outer
loop (``_diloco_ref``): the averaged pseudo-gradient bit for bit from each replica's weights at prepare time, the outer
step within ``outer_ref``'s per-element bound from the device's own state, bit-identical global weights and momentum
on every replica after each commit, a vetoed sync rolled back and retried, a late replica healed with the outer
momentum, and no weight outside the synced fragment touched. This supersedes the 2e-2 bound of
``test_diloco_gpu.py``, which compares the flat path with the generic one on a single replica.

All cases run in one batch of three worker processes (``_diloco_replica.py``); the mutants are deliberate defects the
checks must each catch for their own reason."""

from __future__ import annotations

import json
import os
import subprocess
import sys
from typing import Any, Dict, List

import pytest
import torch

import _q8_emulation as E
from _diloco_ref import outer_ref, pseudo_grad_bits
from _fp64 import _report_margins, assert_close_elementwise  # noqa: F401

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(name: str, model: str, replicas: int, quantize: bool, fragments: int, delay: int, alpha: float, mu: float,
          nesterov: bool, dtype: str = "bf16", syncs: int = 4, **extra: Any) -> Dict[str, Any]:
    return dict(name=name, model=model, replicas=replicas, quantize=quantize, fragments=fragments, delay=delay,
                alpha=alpha, mu=mu, nesterov=nesterov, dtype=dtype, syncs=syncs, **extra)


# a pairwise cover of replicas {2, 3} x quantised x fragments {1, 2} x delay {0, 1} x alpha {0, .5, 1} x
# outer optimizer {plain, momentum, Nesterov}, over llama3_tiny (bf16, FlatParams) and packed fp32 / fp16 weights;
# the foreign-weight cases pack bf16 (gap) and fp32 (tail) weights
MATRIX = [
    _case("llama_2r_q_2f_d1_a05_nest", "llama", 2, True, 2, 1, 0.5, 0.9, True),
    _case("llama_3r_2f_d0_a0_mom", "llama", 3, False, 2, 0, 0.0, 0.9, False),
    _case("llama_2r_1f_d0_a1_sgd", "llama", 2, False, 1, 0, 1.0, 0.0, False),
    _case("llama_3r_q_1f_d1_a0_nest", "llama", 3, True, 1, 1, 0.0, 0.9, True),
    _case("f32_2r_2f_d1_a1_nest", "packed", 2, False, 2, 1, 1.0, 0.9, True, dtype="f32"),
    _case("f32_3r_q_1f_d0_a05_mom", "packed", 3, True, 1, 0, 0.5, 0.9, False, dtype="f32"),
    _case("f16_3r_q_2f_d0_a0_sgd", "packed", 3, True, 2, 0, 0.0, 0.0, False, dtype="f16"),
    _case("f16_2r_1f_d1_a05_mom", "packed", 2, False, 1, 1, 0.5, 0.9, False, dtype="f16"),
    # a hot spare: three replicas, two contributors, the average divides by two
    _case("llama_spare_q", "llama", 3, True, 2, 0, 0.0, 0.9, True, spares=True),
    _case("f32_spare", "packed", 3, False, 1, 1, 0.5, 0.9, False, dtype="f32", spares=True),
]
SPECIAL = [
    _case("rollback", "llama", 2, True, 2, 1, 0.0, 0.9, True, syncs=5, fail_at=2),
    _case("heal", "llama", 3, True, 2, 0, 0.0, 0.9, True, syncs=6, join_after=2),
    _case("slow_side_stream", "llama", 2, True, 2, 1, 0.5, 0.9, True, slow=True),
    _case("slow_side_stream_f32", "packed", 2, False, 2, 1, 0.0, 0.0, False, dtype="f32", slow=True),
    _case("foreign_in_gap", "packed_gap", 2, False, 2, 0, 0.0, 0.9, True),
    _case("foreign_in_tail", "packed_tail", 2, True, 2, 0, 0.0, 0.9, False, dtype="f32"),
]
# each mutant, on a case that exercises it, and the check that must catch it
MUTANTS = [
    ("alpha", _case("m_alpha", "llama", 2, False, 2, 0, 0.0, 0.9, True, mutant="alpha"), "outer step"),
    ("heal_without_momentum", _case("m_heal", "llama", 3, True, 2, 0, 0.0, 0.9, True, syncs=6, join_after=2,
                                    mutant="heal_without_momentum"), "replica agreement"),
    ("world_scale", _case("m_world", "packed", 3, False, 1, 0, 0.0, 0.9, False, dtype="f32", spares=True,
                          mutant="world_scale"), "pseudo-gradient"),
    ("race", _case("m_race", "llama", 2, True, 2, 1, 0.5, 0.9, True, slow=True, mutant="race"), "pseudo-gradient"),
    ("span", _case("m_span", "packed_gap", 2, False, 2, 0, 0.0, 0.9, True, mutant="span"), "ownership"),
]
CASES = MATRIX + SPECIAL + [c for _, c, _ in MUTANTS]


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """Every case, in one batch of three replica processes. Returns the output directory and each process's log."""
    from torchft_b200.bench_utils import local_lighthouse, loopback

    out = tmp_path_factory.mktemp("diloco_exact")
    houses = []
    try:
        cases = []
        for c in CASES:
            lh = local_lighthouse(min_replicas=2 if c.get("join_after") is not None else c["replicas"])
            houses.append(lh)
            cases.append({**c, "lighthouse": loopback(lh.address())})
        spec = out / "cases.json"
        spec.write_text(json.dumps(cases))
        logs = [out / f"replica{r}.log" for r in range(3)]
        procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "_diloco_replica.py"), "--replica", str(r),
                                   "--cases", str(spec), "--out", str(out)], stdout=open(logs[r], "w"),
                                  stderr=subprocess.STDOUT) for r in range(3)]
        for p in procs:
            try:
                p.wait(timeout=900)
            except subprocess.TimeoutExpired:
                p.kill()
                p.wait()
    finally:
        for lh in houses:
            lh.shutdown()
    return out, [log.read_text() for log in logs]


def _load(runs, case: Dict[str, Any]) -> List[List[Dict[str, Any]]]:
    out, logs = runs
    cdir = out / case["name"]
    per = []
    for r in range(case["replicas"]):
        meta_path = cdir / f"r{r}.json"
        assert meta_path.exists(), f"{case['name']}: replica {r} left no records; worker log:\n{logs[r][-6000:]}"
        meta = json.loads(meta_path.read_text())
        recs = [torch.load(cdir / f"r{r}_{k}.pt") for k in range(meta["syncs"])]
        for rec in recs:
            rec["meta"] = meta
        per.append(recs)
    return per


def _first_diff(got: torch.Tensor, want: torch.Tensor) -> str:
    return E.first_mismatch(got, want)


def _bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def check(per: List[List[Dict[str, Any]]], case: Dict[str, Any]) -> None:
    """Every assertion names its check first: pseudo-gradient, outer step, replica agreement, rollback, ownership, heal."""
    name = case["name"]
    # one key per sync: (committed step at prepare, attempt), the same on every replica that took part
    by_key: Dict[Any, Dict[int, Dict[str, Any]]] = {}
    for r, recs in enumerate(per):
        seen: Dict[int, int] = {}
        for k, rec in enumerate(recs):
            attempt = seen.get(rec["step"], 0)
            seen[rec["step"]] = attempt + 1
            rec["replica"], rec["sync"] = r, k
            by_key.setdefault((rec["step"], attempt), {})[r] = rec
    assert by_key, f"{name}: no syncs recorded"
    for key, recs in sorted(by_key.items()):
        frags = {rec["fragment"] for rec in recs.values()}
        assert len(frags) == 1, f"schedule: {name} sync {key}: replicas prepared different fragments {frags}"
        frag = frags.pop()
        where = f"{name} step {key[0]} attempt {key[1]} fragment {frag}"
        verdicts = {rec["verdict"] for rec in recs.values()}
        assert len(verdicts) == 1, f"replica agreement: {where}: verdicts differ"
        verdict = verdicts.pop()
        flat = [rec for rec in recs.values() if rec.get("grad") is not None]
        dtype = next(iter(recs.values()))["storage_before"].dtype

        # pseudo-gradient: bit for bit from the prepare-time snapshots of every replica, in process-group rank order
        if flat:
            ranked = sorted(recs.values(), key=lambda rec: rec["pg_rank"])
            assert [rec["pg_rank"] for rec in ranked] == list(range(ranked[0]["pg_world"])), f"pseudo-gradient: {where}: ranks"
            want = pseudo_grad_bits([rec["snap_orig"] for rec in ranked], [rec["snap_param"] for rec in ranked], dtype,
                                    case["quantize"], [rec["participating"] for rec in ranked], ranked[0]["participants"])
            for rec in flat:
                assert _bits_equal(rec["grad"], want), (
                    f"pseudo-gradient: {where} replica {rec['replica']} sync {rec['sync']}: {_first_diff(rec['grad'], want)}")

        for rec in flat:
            tag = f"{where} replica {rec['replica']} sync {rec['sync']}"
            if verdict:
                # outer step: within outer_ref's bound, from the device's own state before the kernel
                ref = outer_ref(rec["orig_before"], rec["param_before"], rec["mom_before"], rec["grad"], 0.7, case["mu"],
                                case["nesterov"], case["alpha"])
                if ref.mom_slack is None:
                    assert _bits_equal(rec["mom_after"], rec["mom_before"]), f"outer step: {tag}: momentum changed without mu"
                else:
                    assert_close_elementwise(rec["mom_after"], ref.mom, ulps=0, abs_slack=ref.mom_slack,
                                             what=f"outer step: momentum {tag}")
                assert_close_elementwise(rec["orig_after"], ref.orig, ulps=1, abs_slack=ref.orig_slack,
                                         what=f"outer step: global weights {tag}")
                assert_close_elementwise(rec["param_after"], ref.param, ulps=1, abs_slack=ref.param_slack,
                                         what=f"outer step: weights {tag}")
            else:
                # rollback: back to the last global weights, nothing else moves
                assert _bits_equal(rec["param_after"], rec["orig_before"]), (
                    f"rollback: {tag}: weights are not the last global ones: "
                    f"{_first_diff(rec['param_after'], rec['orig_before'])}")
                assert _bits_equal(rec["orig_after"], rec["orig_before"]), f"rollback: {tag}: global weights moved"
                assert _bits_equal(rec["mom_after"], rec["mom_before"]), f"rollback: {tag}: momentum moved"

        # replica agreement: after a commit every replica holds the same global weights and momentum (and the same
        # weights when alpha is 0: they are then the global ones)
        if verdict and len(flat) > 1:
            first = flat[0]
            fields = ["orig_after", "mom_after"] + (["param_after"] if case["alpha"] == 0.0 else [])
            for rec in flat[1:]:
                for f in fields:
                    assert _bits_equal(rec[f], first[f]), (
                        f"replica agreement: {where}: {f} of replica {rec['replica']} (sync {rec['sync']}) differs from "
                        f"replica {first['replica']}: {_first_diff(rec[f], first[f])}")

        # ownership: outside the synced fragment's own weights (padding excluded) no element changes
        for rec in recs.values():
            mask = torch.zeros(rec["storage_before"].numel(), dtype=torch.bool)
            for off, n, fi in rec["meta"]["table"]:
                if fi != frag:
                    mask[off:off + n] = True
            before, after = rec["storage_before"][mask], rec["storage_after"][mask]
            if not _bits_equal(before, after):
                idx = mask.nonzero().flatten()
                bad = int(idx[(before.view(torch.uint8).view(before.numel(), -1)
                               != after.view(torch.uint8).view(after.numel(), -1)).any(1)][0])
                owner = next(fi for off, n, fi in rec["meta"]["table"] if off <= bad < off + n)
                raise AssertionError(
                    f"ownership: {where} replica {rec['replica']} sync {rec['sync']}: storage element {bad} (a weight of "
                    f"fragment {owner}) changed from {rec['storage_before'][bad].item()!r} to "
                    f"{rec['storage_after'][bad].item()!r}")

    # rollback: the window after a vetoed sync retries the same fragment
    for recs in per:
        for a, b in zip(recs, recs[1:]):
            if not a["verdict"]:
                assert b["fragment"] == a["fragment"], f"rollback: {name} replica {a['replica']}: next window synced {b['fragment']}"


@pytest.mark.parametrize("case", MATRIX + SPECIAL, ids=lambda c: c["name"])
def test_flat_diloco_sync_matches_replay(runs, case):
    per = _load(runs, case)
    check(per, case)
    metas = [recs[0]["meta"] for recs in per]
    if case["model"] in ("llama", "packed"):
        assert all(all(m["flat"]) for m in metas)  # the flat path, not the generic fall-back
    if case["model"] == "packed_gap":
        assert not any(metas[0]["flat"]), "a fragment whose span holds another fragment's weight must not be flat"
    if case["model"] == "packed_tail":
        assert metas[0]["flat"] == [False, True], metas[0]["flat"]
    if case.get("fail_at") is not None:
        verdicts = [rec["verdict"] for rec in per[0]]
        assert verdicts.count(False) == 1 and len(verdicts) == case["syncs"] + 1, verdicts
    if case.get("join_after") is not None:
        # heal: the late replica heals, then takes part in at least two committed syncs
        late = per[2]
        assert late and late[0]["step"] >= case["join_after"], [r["step"] for r in late]
        assert sum(rec["verdict"] for rec in late) >= 2, [r["step"] for r in late]
    if case.get("spares"):
        assert [rec["participating"] for recs in per for rec in recs[:1]].count(False) == 1


@pytest.mark.parametrize("mutant,case,caught_by", MUTANTS, ids=[m for m, _, _ in MUTANTS])
def test_mutant_is_caught(runs, mutant, case, caught_by):
    """A deliberate defect makes the checks fail, and for its own reason."""
    per = _load(runs, case)
    with pytest.raises(AssertionError, match=f"^{caught_by}: "):
        check(per, case)
