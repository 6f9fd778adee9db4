"""Spec tests for the C++ control plane.

The scenario tables re-create the reference's Rust unit tests
(upstream src/lighthouse.rs:627-1111, src/manager.rs:656-1218) against
our implementation through the pybind11 module: pure decision functions first,
then real servers on loopback (port 0) driven by real clients.
"""

import os
import threading
import time
import urllib.request
from datetime import timedelta

import pytest

from torchft_b200 import _C

HOUR = 60 * 60 * 1000


def member(rid, step=1, shrink_only=False, commit_failures=0, address="", store=""):
    return _C.QuorumMember(replica_id=rid, address=address, store_address=store, step=step, world_size=1,
                           shrink_only=shrink_only, commit_failures=commit_failures)


def quorum_of(ids, quorum_id=1, steps=None):
    q = _C.Quorum()
    q.quorum_id = quorum_id
    q.participants = [member(i, step=(steps or {}).get(i, 1)) for i in ids]
    return q


# --------------------------------------------------------------- quorum_compute
def test_quorum_join_timeout():
    now = 10 * HOUR * 10
    kw = dict(min_replicas=1, join_timeout_ms=HOUR, heartbeat_timeout_ms=5000)
    met, reason = _C.quorum_compute(now, [], {}, None, **kw)
    assert met is None
    assert "New quorum not ready, only have 0 participants, need min_replicas 1 [0/0 participants healthy]" in reason

    parts = [(now, member("a")), (now, member("b"))]
    hb = {"a": now, "b": now}
    met, reason = _C.quorum_compute(now, parts, hb, None, **kw)
    assert met is not None, reason

    hb["c"] = now  # healthy but not participating -> wait for it
    met, reason = _C.quorum_compute(now, parts, hb, None, **kw)
    assert met is None and "join timeout" in reason

    parts[0] = (now - 10 * HOUR, member("a"))  # first joiner waited long enough
    met, reason = _C.quorum_compute(now, parts, hb, None, **kw)
    assert met is not None, reason
    assert [m.replica_id for m in met] == ["a", "b"]


def test_quorum_heartbeats():
    now = 100 * HOUR
    kw = dict(min_replicas=1, join_timeout_ms=0, heartbeat_timeout_ms=5000)
    parts = [(now, member("a"))]
    met, reason = _C.quorum_compute(now, parts, {"a": now}, None, **kw)
    assert met is not None
    assert "[1/1 participants healthy][1 heartbeating]" in reason

    met, reason = _C.quorum_compute(now, parts, {"a": now - 10_000}, None, **kw)  # expired
    assert met is None
    assert "[0/1 participants healthy][0 heartbeating]" in reason

    parts.append((now, member("b")))
    met, reason = _C.quorum_compute(now, parts, {"a": now - 10_000, "b": now}, None, **kw)
    assert met is not None, reason
    assert [m.replica_id for m in met] == ["b"]


def test_quorum_fast_prev_quorum():
    now = 100 * HOUR
    kw = dict(min_replicas=1, join_timeout_ms=HOUR, heartbeat_timeout_ms=5000)
    parts = [(now, member("a"))]
    hb = {"a": now, "b": now}
    met, reason = _C.quorum_compute(now, parts, hb, None, **kw)
    assert met is None, reason  # b heartbeats but has not joined; join timeout not reached

    prev = quorum_of(["a"])
    met, reason = _C.quorum_compute(now, parts, hb, prev, **kw)
    assert met is not None and "Fast quorum found" in reason

    # fast quorum may also grow
    parts.append((now, member("b")))
    met, reason = _C.quorum_compute(now, parts, hb, prev, **kw)
    assert met is not None and [m.replica_id for m in met] == ["a", "b"]


def test_quorum_shrink_only():
    now = 100 * HOUR
    kw = dict(min_replicas=1, join_timeout_ms=HOUR, heartbeat_timeout_ms=5000)
    prev = quorum_of(["a", "b"])
    parts = [(now, member("a", shrink_only=True)), (now, member("c", shrink_only=True))]
    hb = {"a": now, "c": now}
    met, reason = _C.quorum_compute(now, parts, hb, prev, **kw)
    assert met is not None, reason
    assert "[shrink_only=true]" in reason
    assert [m.replica_id for m in met] == ["a"]


def test_quorum_split_brain():
    now = 100 * HOUR
    kw = dict(min_replicas=1, join_timeout_ms=HOUR, heartbeat_timeout_ms=5000)
    parts = [(now - 2 * HOUR, member("a"))]
    hb = {"a": now, "b": now}
    met, reason = _C.quorum_compute(now, parts, hb, None, **kw)
    assert met is None
    assert "New quorum not ready, only have 1 participants, need at least half of 2 healthy workers" in reason
    parts.append((now - 2 * HOUR, member("b")))
    met, reason = _C.quorum_compute(now, parts, hb, None, **kw)
    assert met is not None, reason


def test_quorum_changed():
    a, b, c = member("1"), member("1"), member("2")
    a.address, b.address = "x", "y"  # only ids matter
    assert not _C.quorum_changed([a], [b])
    assert _C.quorum_changed([a], [c])
    assert _C.quorum_changed([a], [a, c])


# --------------------------------------------------------- compute_quorum_results
def _q(steps, commit_failures=None):
    q = _C.Quorum()
    q.quorum_id = 1
    q.participants = [
        member(f"replica_{i}", step=s, address=f"addr_{i}", store=f"store_addr_{i}",
               commit_failures=(commit_failures or {}).get(i, 0))
        for i, s in enumerate(steps)
    ]
    return q


def test_compute_quorum_results_first_step():
    q = _q([0, 0])
    r = _C.compute_quorum_results("replica_0", 0, q, True)
    assert (r.heal, r.replica_rank, r.recover_src_replica_rank, r.recover_dst_replica_ranks) == (False, 0, None, [1])
    r = _C.compute_quorum_results("replica_1", 0, q, True)
    assert (r.heal, r.replica_rank, r.recover_src_replica_rank, r.recover_dst_replica_ranks) == (True, 1, 0, [])
    # shard rank 1 rotates the primary
    r = _C.compute_quorum_results("replica_1", 1, q, True)
    assert (r.heal, r.replica_rank, r.recover_src_replica_rank, r.recover_dst_replica_ranks) == (False, 1, None, [0])
    assert r.store_address == "store_addr_1"


def test_compute_quorum_results_recovery():
    q = _q([0, 1, 0, 1, 0])
    r = _C.compute_quorum_results("replica_0", 0, q, True)
    assert r.heal and r.recover_src_manager_address == "addr_1" and r.recover_src_replica_rank == 1
    assert r.recover_dst_replica_ranks == [] and r.max_step == 1 and r.max_world_size == 2
    assert r.max_replica_rank is None and r.replica_world_size == 5
    r = _C.compute_quorum_results("replica_1", 0, q, True)
    assert not r.heal and r.recover_src_manager_address == "" and r.recover_dst_replica_ranks == [0, 4]
    assert r.max_replica_rank == 0
    r = _C.compute_quorum_results("replica_3", 0, q, True)
    assert not r.heal and r.replica_rank == 3 and r.recover_dst_replica_ranks == [2] and r.max_replica_rank == 1
    r = _C.compute_quorum_results("replica_1", 1, q, True)
    assert not r.heal and r.recover_dst_replica_ranks == [2]
    assert r.replica_ids == [f"replica_{i}" for i in range(5)]


def test_compute_quorum_results_skip_init_sync():
    q = _q([0, 0])
    assert not _C.compute_quorum_results("replica_0", 0, q, True).heal
    assert _C.compute_quorum_results("replica_1", 0, q, True).heal
    assert not _C.compute_quorum_results("replica_1", 0, q, False).heal
    q = _q([1, 0])
    assert _C.compute_quorum_results("replica_1", 0, q, False).heal


def test_compute_quorum_results_commit_failures_and_missing():
    q = _q([0, 0], commit_failures={1: 2})
    assert _C.compute_quorum_results("replica_0", 0, q, True).commit_failures == 2
    with pytest.raises(RuntimeError, match="not participating"):
        _C.compute_quorum_results("nope", 0, q, True)


def test_backoff_schedule():
    s = _C.backoff_schedule(20)
    assert s[0] == 100 and abs(s[1] - 150) < 1e-6 and abs(s[2] - 225) < 1e-6
    assert max(s) == 10000 and s == sorted(s)


# ----------------------------------------------------------------- real servers
@pytest.fixture
def lighthouse():
    lh = _C.LighthouseServer(bind="[::]:0", min_replicas=1, join_timeout_ms=100, quorum_tick_ms=10)
    yield lh
    lh.shutdown()


def test_lighthouse_e2e(lighthouse):
    c = _C.LighthouseClient(lighthouse.address(), timedelta(seconds=5))
    c.heartbeat("foo")
    t0 = time.time()
    q = c.quorum("foo", timedelta(seconds=5), address="addr", store_address="store", step=10, world_size=1,
                 data={"k": [1, 2]})
    assert time.time() - t0 < 0.4  # single replica join < 0.4 s (reference: lighthouse_test.py:50-53)
    assert q.quorum_id == 1 and len(q.participants) == 1
    p = q.participants[0]
    assert (p.replica_id, p.address, p.store_address, p.step, p.world_size) == ("foo", "addr", "store", 10, 1)
    assert p.data == {"k": [1, 2]}
    assert q.created.seconds > 1_600_000_000
    # same membership -> same id
    assert c.quorum("foo", timedelta(seconds=5)).quorum_id == 1


def test_lighthouse_timeout_and_runtime_errors():
    lh = _C.LighthouseServer(bind="[::]:0", min_replicas=2, join_timeout_ms=100)
    try:
        c = _C.LighthouseClient(lh.address(), timedelta(seconds=5))
        t0 = time.time()
        with pytest.raises(TimeoutError):
            c.quorum("lonely", timedelta(milliseconds=200))
        assert time.time() - t0 < 1.0
    finally:
        lh.shutdown()
    with pytest.raises(TimeoutError):
        _C.LighthouseClient("http://localhost:1", timedelta(milliseconds=300))


def test_lighthouse_join_during_shrink():
    """A joiner is excluded from a shrink_only round and admitted to the next one."""
    lh = _C.LighthouseServer(bind="[::]:0", min_replicas=2, join_timeout_ms=1000, quorum_tick_ms=10)
    try:
        addr = lh.address()
        c0 = _C.LighthouseClient(addr, timedelta(seconds=5))
        c1 = _C.LighthouseClient(addr, timedelta(seconds=5))
        c2 = _C.LighthouseClient(addr, timedelta(seconds=5))
        out = {}

        def ask(name, client, **kw):
            out[name] = client.quorum(name, timedelta(seconds=10), **kw)

        ts = [threading.Thread(target=ask, args=("replica0", c0)), threading.Thread(target=ask, args=("replica1", c1))]
        [t.start() for t in ts]
        [t.join() for t in ts]
        assert out["replica0"].quorum_id == out["replica1"].quorum_id == 1
        assert len(out["replica0"].participants) == 2

        # shrink round: replica0 asks shrink_only while replica2 tries to join
        t2 = threading.Thread(target=ask, args=("replica2", c2))
        t2.start()
        time.sleep(0.1)
        ts = [threading.Thread(target=ask, args=("replica0", c0), kwargs=dict(shrink_only=True)),
              threading.Thread(target=ask, args=("replica1", c1))]
        [t.start() for t in ts]
        [t.join() for t in ts]
        ids = sorted(p.replica_id for p in out["replica0"].participants)
        assert ids == ["replica0", "replica1"], ids
        assert out["replica0"].quorum_id == 1  # membership unchanged -> id unchanged

        # next (non-shrink) round admits replica2 and bumps the id
        ts = [threading.Thread(target=ask, args=("replica0", c0)), threading.Thread(target=ask, args=("replica1", c1))]
        [t.start() for t in ts]
        [t.join() for t in ts]
        t2.join()
        assert sorted(p.replica_id for p in out["replica2"].participants) == ["replica0", "replica1", "replica2"]
        assert out["replica2"].quorum_id == 2
    finally:
        lh.shutdown()


def test_lighthouse_commit_failures_bump_quorum_id(lighthouse):
    lhc = _C.LighthouseClient(lighthouse.address(), timedelta(seconds=5))
    assert lhc.quorum("r", timedelta(seconds=5)).quorum_id == 1
    assert lhc.quorum("r", timedelta(seconds=5)).quorum_id == 1
    # commit failures travel through the manager path
    ms = _C.ManagerServer(replica_id="r", lighthouse_addr=lighthouse.address(), hostname="localhost", bind="[::]:0",
                          store_addr="s", world_size=1, heartbeat_interval=timedelta(milliseconds=50),
                          connect_timeout=timedelta(seconds=5), quorum_retries=0)
    try:
        mc = _C.ManagerClient(ms.address(), timedelta(seconds=5))
        a = mc._quorum(0, 0, "", False, timedelta(seconds=5), 0)
        b = mc._quorum(0, 0, "", False, timedelta(seconds=5), 0)
        assert a.quorum_id == b.quorum_id
        c = mc._quorum(0, 0, "", False, timedelta(seconds=5), 2)
        assert c.quorum_id == b.quorum_id + 1 and c.commit_failures == 2
    finally:
        ms.shutdown()


def _manager(lh, rid, world_size=1, **kw):
    return _C.ManagerServer(replica_id=rid, lighthouse_addr=lh.address(), hostname="localhost", bind="[::]:0",
                            store_addr=f"store_{rid}", world_size=world_size,
                            heartbeat_interval=timedelta(milliseconds=50), connect_timeout=timedelta(seconds=5),
                            quorum_retries=kw.get("quorum_retries", 0))


def test_manager_should_commit_barrier(lighthouse):
    ms = _manager(lighthouse, "rep", world_size=2)
    try:
        def vote(rank, v, out):
            c = _C.ManagerClient(ms.address(), timedelta(seconds=5))
            out[rank] = c.should_commit(rank, 1, v, timedelta(seconds=5))

        for votes, expect in (((True, True), True), ((True, False), False), ((True, True), True)):
            out = {}
            ts = [threading.Thread(target=vote, args=(r, v, out)) for r, v in enumerate(votes)]
            [t.start() for t in ts]
            [t.join() for t in ts]
            assert out == {0: expect, 1: expect}
        # a lone voter times out quickly (reference asserts < 1.0 s: manager_integ_test.py:555-567)
        c = _C.ManagerClient(ms.address(), timedelta(seconds=5))
        t0 = time.time()
        with pytest.raises(TimeoutError):
            c.should_commit(0, 1, True, timedelta(milliseconds=100))
        assert time.time() - t0 < 1.0
    finally:
        ms.shutdown()


def test_manager_quorum_heal_first_step_and_metadata():
    # min_replicas=2: the quorum must contain BOTH groups no matter how the two requests are scheduled
    lighthouse = _C.LighthouseServer(bind="[::]:0", min_replicas=2, join_timeout_ms=100, quorum_tick_ms=10)
    m0, m1 = _manager(lighthouse, "rep_0"), _manager(lighthouse, "rep_1")
    try:
        res = {}

        def run(i, m, step):
            c = _C.ManagerClient(m.address(), timedelta(seconds=5))
            res[i] = c._quorum(0, step, f"meta_{i}", False, timedelta(seconds=10), 0, True)

        ts = [threading.Thread(target=run, args=(0, m0, 0)), threading.Thread(target=run, args=(1, m1, 0))]
        [t.start() for t in ts]
        [t.join() for t in ts]
        assert res[0].replica_rank == 0 and not res[0].heal and res[0].recover_dst_replica_ranks == [1]
        assert res[1].replica_rank == 1 and res[1].heal and res[1].recover_src_replica_rank == 0
        assert res[1].recover_src_manager_address == m0.address()
        assert res[0].store_address == res[1].store_address == "store_rep_0"
        assert res[0].replica_ids == ["rep_0", "rep_1"]
        # healer looks up the source's transport metadata through the source's manager
        c = _C.ManagerClient(res[1].recover_src_manager_address, timedelta(seconds=5))
        assert c._checkpoint_metadata(0, timedelta(seconds=5)) == "meta_0"
        with pytest.raises(RuntimeError, match="rank not found"):
            c._checkpoint_metadata(7, timedelta(seconds=5))
    finally:
        m0.shutdown()
        m1.shutdown()
        lighthouse.shutdown()


def test_manager_quorum_group_barrier_times_out(lighthouse):
    ms = _manager(lighthouse, "rep", world_size=2)
    try:
        c = _C.ManagerClient(ms.address(), timedelta(seconds=5))
        t0 = time.time()
        with pytest.raises(TimeoutError):
            c._quorum(0, 0, "", False, timedelta(milliseconds=100), 0)
        assert time.time() - t0 < 1.0
    finally:
        ms.shutdown()


def test_manager_survives_lighthouse_restart_with_retries():
    lh = _C.LighthouseServer(bind="[::]:0", min_replicas=1, join_timeout_ms=100)
    addr = lh.address()
    port = int(addr.rsplit(":", 1)[1])
    ms = _C.ManagerServer(replica_id="rep", lighthouse_addr=addr, hostname="localhost", bind="[::]:0",
                          store_addr="s", world_size=1, heartbeat_interval=timedelta(milliseconds=50),
                          connect_timeout=timedelta(seconds=3), quorum_retries=8)
    try:
        c = _C.ManagerClient(ms.address(), timedelta(seconds=5))
        assert c._quorum(0, 0, "", False, timedelta(seconds=5), 0).quorum_id == 1
        lh.shutdown()
        box = {}

        def ask():
            try:
                box["r"] = c._quorum(0, 1, "", False, timedelta(seconds=8), 0)
            except Exception as e:  # pragma: no cover
                box["e"] = e

        t = threading.Thread(target=ask)
        t.start()
        time.sleep(0.5)
        lh = _C.LighthouseServer(bind=f"[::]:{port}", min_replicas=1, join_timeout_ms=100)
        t.join()
        assert "r" in box, box
        assert box["r"].replica_world_size == 1
    finally:
        ms.shutdown()
        lh.shutdown()


def test_manager_quorum_fails_fast_when_lighthouse_down():
    lh = _C.LighthouseServer(bind="[::]:0", min_replicas=1, join_timeout_ms=100)
    ms = _C.ManagerServer(replica_id="rep", lighthouse_addr=lh.address(), hostname="localhost", bind="[::]:0",
                          store_addr="s", world_size=1, heartbeat_interval=timedelta(milliseconds=50),
                          connect_timeout=timedelta(milliseconds=200), quorum_retries=0)
    try:
        lh.shutdown()
        c = _C.ManagerClient(ms.address(), timedelta(seconds=5))
        t0 = time.time()
        with pytest.raises((RuntimeError, TimeoutError)):
            c._quorum(0, 0, "", False, timedelta(seconds=5), 0)
        assert time.time() - t0 < 4.0  # error is broadcast, waiters do not hang to their deadline
    finally:
        ms.shutdown()


def test_dashboard_http(lighthouse):
    c = _C.LighthouseClient(lighthouse.address(), timedelta(seconds=5))
    c.quorum("dash", timedelta(seconds=5), address="http://nowhere:1", step=4)
    port = lighthouse.address().rsplit(":", 1)[1]
    index = urllib.request.urlopen(f"http://127.0.0.1:{port}/").read().decode()
    assert "Lighthouse" in index and "/status" in index
    status = urllib.request.urlopen(f"http://127.0.0.1:{port}/status").read().decode()
    assert "dash" in status and "Step: 4" in status and "Heartbeats" in status
    with pytest.raises(urllib.error.HTTPError):
        urllib.request.urlopen(urllib.request.Request(f"http://127.0.0.1:{port}/replica/nobody/kill", method="POST"))


@pytest.mark.parametrize("sanitize,needle", [("thread", "ThreadSanitizer"), ("address", "Sanitizer")])
def test_native_selftest_under_sanitizers(sanitize, needle):
    """Race detection / memory checking of the C++ control plane: the same selftest under TSan and ASan+UBSan.
    (TSan found a real bug in round 1: a worker thread notified a condition variable after the server that owned
    it could already be destroyed.)"""
    import subprocess

    from torchft_b200 import _build

    try:
        exe = _build.build_selftest(sanitize=sanitize)
    except Exception as e:  # noqa: BLE001 - toolchain without the sanitizer runtime
        pytest.skip(f"cannot build with -fsanitize={sanitize}: {e}")
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 second_deadlock_stack=1", ASAN_OPTIONS="detect_leaks=1",
               UBSAN_OPTIONS="print_stacktrace=1")
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300, env=env)
    out = r.stdout + r.stderr
    if "selftest:" not in r.stdout and ("unexpected memory mapping" in out or "Shadow memory" in out or "ReserveShadowMemoryRange" in out):
        pytest.skip(f"{sanitize} sanitizer runtime cannot start in this environment (ASLR / address-space layout)")
    assert "0 failed" in r.stdout, out[-3000:]
    assert needle not in out and "runtime error" not in out, out[-4000:]
    assert r.returncode == 0


def test_restarted_lighthouse_never_reuses_quorum_ids():
    """quorum_id_base=-1 (CLI: --quorum_id_base auto): ids come from the clock, so a new incarnation starts above
    everything the previous one handed out (process groups rendezvous under store prefixes keyed by quorum id)."""
    ids = []
    for _ in range(2):
        lh = _C.LighthouseServer(bind="[::]:0", min_replicas=1, join_timeout_ms=50, quorum_tick_ms=10, quorum_id_base=-1)
        try:
            c = _C.LighthouseClient(lh.address(), timedelta(seconds=5))
            first = c.quorum("a", timedelta(seconds=5)).quorum_id
            # membership change -> bump
            import threading

            t = threading.Thread(target=lambda: _C.LighthouseClient(lh.address(), timedelta(seconds=5)).quorum("b", timedelta(seconds=5)))
            t.start()
            from torchft_b200.coordination import lighthouse_status

            deadline = time.time() + 5  # "b" alone is not a majority of {a, b}: it waits until "a" asks again
            while "b" not in lighthouse_status(lh.address().replace("[::]", "127.0.0.1"))["waiting"]:
                assert time.time() < deadline
                time.sleep(0.01)
            second = c.quorum("a", timedelta(seconds=5)).quorum_id
            t.join()
            assert second == first + 1
            ids += [first, second]
        finally:
            lh.shutdown()
        time.sleep(0.6)
    assert ids == sorted(ids) and len(set(ids)) == 4 and ids[2] > ids[1]
    assert ids[0] < 2 ** 31  # fits the 32-bit epoch field of the in-kernel flags
    # default stays reference-compatible: first quorum has id 1
    lh = _C.LighthouseServer(bind="[::]:0", min_replicas=1, join_timeout_ms=50)
    try:
        assert _C.LighthouseClient(lh.address(), timedelta(seconds=5)).quorum("a", timedelta(seconds=5)).quorum_id == 1
    finally:
        lh.shutdown()


def test_status_json(lighthouse):
    import json

    c = _C.LighthouseClient(lighthouse.address(), timedelta(seconds=5))
    c.quorum('we"ird\\id', timedelta(seconds=5), address="http://nowhere:1", store_address="s:1", step=9, world_size=2)
    port = lighthouse.address().rsplit(":", 1)[1]
    r = urllib.request.urlopen(f"http://127.0.0.1:{port}/status.json")
    assert r.headers["Content-Type"].startswith("application/json")
    st = json.loads(r.read().decode())
    assert st["quorum_id"] >= 1 and st["prev_quorum"]["max_step"] == 9
    (p,) = st["prev_quorum"]["participants"]
    assert p["replica_id"] == 'we"ird\\id' and p["step"] == 9 and p["world_size"] == 2 and p["recovering"] is False
    assert st["heartbeats"]['we"ird\\id']["alive"] is True
    assert isinstance(st["next_quorum_status"], str) and st["min_replicas"] == 1


def test_native_selftest_binary():
    """The C++ control plane's own unit + integration tests (the reference runs `cargo test`)."""
    import subprocess

    from torchft_b200 import _build

    exe = _build.build_selftest()
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 failed" in r.stdout


def test_server_survives_malformed_traffic(lighthouse):
    """Garbage, truncated frames, absurd lengths, unknown methods and undecodable payloads must never take the
    Lighthouse down or wedge it (the reference gets this from tonic/hyper; our framing is hand-written)."""
    import os
    import socket
    import struct

    port = int(lighthouse.address().rsplit(":", 1)[1])

    def raw(data: bytes, read: bool = True, linger: float = 0.2) -> bytes:
        s = socket.create_connection(("127.0.0.1", port), timeout=5)
        try:
            s.sendall(data)
            if not read:
                return b""
            s.settimeout(linger)
            try:
                return s.recv(65536)
            except (socket.timeout, ConnectionResetError):
                return b""
        finally:
            s.close()

    def frame(method: int, payload: bytes, timeout_ms: int = 1000, length: int = -1) -> bytes:
        return b"TFT1" + struct.pack("<IQI", method, timeout_ms, len(payload) if length < 0 else length) + payload

    rng_bytes = os.urandom(4096)
    raw(rng_bytes)                                     # not our magic, not HTTP
    raw(b"GET /nope HTTP/1.1\r\n\r\n")                 # unknown HTTP path -> 404
    raw(b"GET " + b"A" * 100000)                       # endless request line, never terminated
    raw(b"TFT", read=False)                            # truncated magic, then EOF
    raw(b"TFT1" + b"\x01\x00", read=False)             # truncated header
    raw(frame(1, b"\x00" * 10, length=1 << 31), read=False)      # claims 2 GiB: must be refused, not allocated
    raw(frame(1, b"\x00" * 10, length=5000), read=False)         # claims more than it sends, then EOF
    for method in (0, 7, 999, 2 ** 32 - 1):            # unknown methods -> error status, connection stays sane
        resp = raw(frame(method, b"hello"))
        assert len(resp) >= 8 and struct.unpack("<I", resp[:4])[0] != 0
    for method in (1, 2):                              # known methods, undecodable payloads
        for payload in (b"", b"\xff" * 3, rng_bytes[:64], struct.pack("<I", 2 ** 31) + b"x"):
            resp = raw(frame(method, payload))
            assert len(resp) >= 8 and struct.unpack("<I", resp[:4])[0] != 0, (method, payload[:8])
    # ... and it still does its job
    c = _C.LighthouseClient(lighthouse.address(), timedelta(seconds=5))
    q = c.quorum("after_fuzz", timedelta(seconds=5), address="http://x:1", step=1)
    assert [p.replica_id for p in q.participants] == ["after_fuzz"]
    c.heartbeat("after_fuzz", timedelta(seconds=1))
    status = urllib.request.urlopen(f"http://127.0.0.1:{port}/status.json").read()
    assert b"after_fuzz" in status


@pytest.mark.parametrize("how", ["python_module", "standalone_binary"])
def test_lighthouse_command_line(how):
    """`python -m torchft_b200.lighthouse` and the stand-alone binary take the reference's flags (+ --quorum_id_base),
    serve RPC + dashboard on one port, and stop on SIGINT/SIGTERM."""
    import signal
    import socket
    import subprocess
    import sys

    from torchft_b200 import _build
    from torchft_b200.coordination import wait_for_lighthouse

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    flags = ["--bind", f"127.0.0.1:{port}", "--min_replicas", "3", "--join_timeout_ms", "250", "--quorum_tick_ms", "20",
             "--heartbeat_timeout_ms", "1500", "--quorum_id_base", "auto"]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torchft_b200.lighthouse"] if how == "python_module" else [str(_build.build_lighthouse_binary())]
    p = subprocess.Popen(cmd + flags, cwd=root, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        st = wait_for_lighthouse(f"http://127.0.0.1:{port}", timedelta(seconds=60))
        assert st["min_replicas"] == 3 and st["heartbeat_timeout_ms"] == 1500 and st["quorum_id"] > 10 ** 6  # clock-based base
        c = _C.LighthouseClient(f"http://127.0.0.1:{port}", timedelta(seconds=5))
        c.heartbeat("cli_probe", timedelta(seconds=2))
        with pytest.raises(TimeoutError):
            c.quorum("cli_probe", timedelta(milliseconds=300))  # 1 of min_replicas=3
        p.send_signal(signal.SIGINT if how == "python_module" else signal.SIGTERM)
        assert p.wait(20) is not None
    finally:
        if p.poll() is None:
            p.kill()
    # a missing required flag is a usage error, not a hang
    r = subprocess.run(cmd + ["--bind", "127.0.0.1:0"], cwd=root, capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "min_replicas" in (r.stdout + r.stderr)
