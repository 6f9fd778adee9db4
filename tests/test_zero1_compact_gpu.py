"""FT-ZeRO-1 compact (paged) optimizer state on ONE GPU: the paged update kernel against the flat one, and a compact
``Zero1Optimizer`` against a full-size one through kills, rejoins and split commits (ranks emulated in-process with
``SymmetricComm.virtual_world``)."""

from __future__ import annotations

import threading
from datetime import timedelta

import pytest
import torch

from _zero1_replicas import HP, NUMEL, SHIFT, UNITS, Replicas, kernel_world
from _zero1_state import State

pytestmark = pytest.mark.gpu


def _run_update_kernels(world, k, presignal, paged, seed):
    """Several gated steps (one vetoed), then a refresh, on fresh ranks; returns the weights and the state of every rank
    as full-size tensors (paged state gathered back through its page table)."""
    dev = torch.device("cuda", 0)
    comms = kernel_world(world, presignal)
    g = torch.Generator(device=dev).manual_seed(seed)
    init = (torch.randn(NUMEL, device=dev, generator=g) * 0.05).bfloat16()
    params = [c.segment("z1_param")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    grads = [torch.empty(NUMEL, dtype=torch.bfloat16, device=dev) for _ in comms]
    state = [State.seeded(init, SHIFT if paged else None, seed * 10 + r) for r in range(world)]
    for p in params:
        p.copy_(init)
    gates = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in comms]
    streams = [torch.cuda.Stream(device=dev) for _ in comms]

    def launch(r, mode, host_ok):
        c, s = comms[r], (streams[r] if not presignal else torch.cuda.current_stream())
        with torch.cuda.stream(s):
            if mode == 0:
                c.zero1_commit_(gates[r], host_ok, True, s)
            for lo, hi in UNITS:
                c.zero1_update_("z1_param", lo * 2, grads[r].data_ptr() + lo * 2, nelem=hi - lo, hyper=HP, gate=gates[r],
                                replication=k, mode=mode, blocks=4, stream=s, **state[r].args(lo))

    for step, (mode, veto) in enumerate([(0, False), (0, False), (0, True), (0, False), (1, False), (0, False)]):
        gstep = torch.randn(NUMEL, device=dev, generator=g).bfloat16()
        for r in range(world):
            grads[r].copy_(gstep)
        torch.cuda.synchronize()
        for r in range(world):
            launch(r, mode, not (veto and r == world - 1))
        torch.cuda.synchronize()
        assert all(c.errored() is None for c in comms)
    return [p.clone() for p in params], [st.get(0, NUMEL) for st in state], [gt.clone() for gt in gates]


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_paged_update_matches_flat_update_bit_for_bit(world, k):
    _check_paged_vs_flat(world, k, presignal=True)


def test_paged_update_matches_flat_update_with_real_signalling():
    """All ranks in flight at once on W streams (presignal off)."""
    _check_paged_vs_flat(4, 2, presignal=False)


def _check_paged_vs_flat(world, k, presignal):
    from torchft_b200.parallel.zero1 import ShardLayout

    L = ShardLayout(tuple(UNITS), k)
    pf, sf, gf = _run_update_kernels(world, k, presignal, False, 7 + world * 3 + k)
    pp, sp, gp = _run_update_kernels(world, k, presignal, True, 7 + world * 3 + k)
    for r in range(world):
        assert torch.equal(gf[r], gp[r])
        assert torch.equal(pf[r], pp[r]), f"weights of rank {r}"
        for lo, hi in L.held(r, world):
            for name, a, b in zip(("master", "m", "v"), sf[r], sp[r]):
                assert torch.equal(a[lo:hi], b[lo:hi]), f"{name} of rank {r} on [{lo}, {hi})"
    # five gated steps; the veto of the last rank reaches everybody only when the ranks really signal each other
    assert int(gf[0][1]) == (5 if presignal else 4) and int(gf[world - 1][1]) == 4


# ----------------------------------------------------------------------------- Zero1Optimizer, compact vs full-size
def test_compact_optimizer_tracks_full_size_optimizer_through_kill_rejoin_and_split_commit():
    import json

    from torch.distributed import PrefixStore

    from torchft_b200.parallel.symm_mem import SymmetricComm
    from torchft_b200.parallel.zero1 import ShardLayout, page_ranges, pool_pages

    dev = torch.device("cuda", 0)
    n, k, min_world = 4, 2, 3
    cap = pool_pages(ShardLayout(tuple(UNITS), k), min_world, 1 << SHIFT)
    assert cap < NUMEL >> SHIFT  # the pools really are smaller than the vector
    g = torch.Generator(device=dev).manual_seed(3)
    init = (torch.randn(NUMEL, device=dev, generator=g) * 0.05).bfloat16()
    reps = {kind: Replicas(n, k=k, compact=kind == "compact", min_world=min_world, init=init)
            for kind in ("flat", "compact")}
    opts = {kind: r.opts for kind, r in reps.items()}
    assert opts["compact"][0].state_bytes_allocated() == 12 * (cap << SHIFT)
    assert opts["flat"][0].state_bytes_allocated() == 12 * NUMEL

    def configure(members, epoch):
        for r in reps.values():
            r.configure(members, epoch)

    def step(members, veto=()):
        gstep = torch.randn(NUMEL, device=dev, generator=g).bfloat16()  # the reduced gradient, identical everywhere
        for r in reps.values():
            r.step([[gstep] * len(members)], veto=veto, reduce=False)
            r.settle()
        for m in members:
            f, c = opts["flat"][m], opts["compact"][m]
            assert f.t == c.t and f._holdings == c._holdings
            assert torch.equal(f.param, c.param), f"weights of member {m}"
            hf, hc = f.held_state(), c.held_state()
            assert hf.keys() == hc.keys()
            for rng in hf:
                for a, b in zip(hf[rng], hc[rng]):
                    assert torch.equal(a, b), f"state of member {m} on {rng}"

    configure([0, 1, 2, 3], 1)
    step([0, 1, 2, 3]); step([0, 1, 2, 3])
    configure([0, 1, 3], 2)                        # kill: 4 -> 3
    assert opts["compact"][0].lost_elements == 0
    step([0, 1, 3])
    for r in reps.values():                        # rejoin: 3 -> 4, member 2 restarts from the healed weights
        o = r.make(r.comms[2])
        o.param.copy_(r.opts[0].param)
        o.seed_master()
        r.opts[2] = o
    configure([0, 1, 2, 3], 3)
    step([0, 1, 2, 3])
    step([0, 1, 2, 3], veto=[1])                   # split commit: member 1 misses the update the others apply
    assert opts["compact"][1].t + 1 == opts["compact"][0].t
    configure([0, 1, 2, 3], 4)
    step([0, 1, 2, 3])
    for m in range(n):
        assert opts["compact"][m].lost_elements == opts["flat"][m].lost_elements == 0
        assert opts["compact"][m].state_bytes_held() == opts["flat"][m].state_bytes_held()
    # a re-shard to [0, 1, 3] that fails at the barrier: member 3 publishes and then dies, members 0 and 1 have already
    # freed and allocated pages. They keep their update count and may claim only ranges their kept pages still back.
    comp_c, c3 = reps["compact"].comms, opts["compact"][3]
    qs = PrefixStore("q/5", reps["compact"].store)
    qs.set("z1/2", json.dumps({"t": c3.t, "hold": c3._holdings, "pages": c3._page_runs()}))
    SymmetricComm.virtual_quorum(comp_c, [0, 1, 3], 5)
    for m in (0, 1):
        comp_c[m]._timeout = timedelta(seconds=1)
    errs = []
    ts = [threading.Thread(target=lambda m=m: errs.append(_raises(opts["compact"][m]._on_configured, qs, m, 3, 5)))
          for m in (0, 1)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert all(isinstance(e, TimeoutError) for e in errs), errs
    for m in (0, 1):
        comp_c[m]._timeout = timedelta(seconds=20)
        o = opts["compact"][m]
        assert o.t == opts["flat"][m].t
        assert all(o._table_host[p] >= 0 for lo, hi in page_ranges(o._holdings, SHIFT) for p in range(lo, hi))
    configure([0, 1, 2, 3], 6)                     # the retry with everybody: nothing is lost, state matches again
    step([0, 1, 2, 3])
    for m in range(n):
        assert opts["compact"][m].lost_elements == 0
    # a quorum below min_world is refused before any state moves
    SymmetricComm.virtual_quorum(comp_c, [0, 1], 7)
    with pytest.raises(RuntimeError, match="min_world"):
        opts["compact"][0]._on_configured(PrefixStore("q/7", reps["compact"].store), 0, 2, 7)


def _raises(fn, *args):
    try:
        fn(*args)
    except Exception as e:  # noqa: BLE001
        return e
    return None
