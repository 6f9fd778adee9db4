"""torchcomms adapter, torchx component, failure injection, local orchestrator."""

from __future__ import annotations

import os
import subprocess
import sys
import threading
import time
from datetime import timedelta

import pytest
import torch
import torch.distributed as dist
from torch.distributed import PrefixStore, TCPStore

from torchft_b200.failure import Failure, FailureInjector, send_failure
from torchft_b200.process_group import FakeProcessGroupWrapper, ProcessGroupDummy
from torchft_b200.torchcomms import ProcessGroupTorchComms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Done:
    def __init__(self, work=None):
        self._w = work

    def wait(self):
        if self._w is not None:
            self._w.wait()

    def is_completed(self):
        return self._w is None or self._w.is_completed()


class _LoopbackComm:
    """A reconfigurable communicator for the adapter test: one long-lived object whose
    membership is swapped by reconfigure() (handles are ``host:port`` of a per-comm store)."""

    def __init__(self):
        self._store = TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)
        self._handle = f"127.0.0.1:{self._store.port}"
        self._pg = None
        self.reconfigures = 0
        self.finalized = False

    def get_backend(self):
        return "loopback-gloo"

    def get_device(self):
        return torch.device("cpu")

    def get_init_handle(self):
        return self._handle

    def reconfigure(self, uuid, init_handles, timeout):
        rank = init_handles.index(self._handle)
        host, port = init_handles[0].rsplit(":", 1)
        root = self._store if rank == 0 else TCPStore(host, int(port), is_master=False, wait_for_workers=False)
        self._pg = dist.ProcessGroupGloo(PrefixStore(f"q{uuid}", root), rank, len(init_handles), timeout)
        self.reconfigures += 1
        return _Done()

    def finalize(self):
        self.finalized = True
        self._pg = None

    def all_reduce(self, t, op, async_op=True):
        o = dist.AllreduceOptions()
        o.reduceOp = op
        return _Done(self._pg.allreduce([t], o))

    def broadcast(self, t, root, async_op=True):
        o = dist.BroadcastOptions()
        o.rootRank = root
        return _Done(self._pg.broadcast([t], o))

    def all_gather(self, outs, t, async_op=True):
        return _Done(self._pg.allgather([outs], [t]))

    def barrier(self, async_op=True):
        return _Done(self._pg.barrier())

    def send(self, t, dst, async_op=True):
        return _Done(self._pg.send([t], dst, 0))

    def recv(self, t, src, async_op=True):
        return _Done(self._pg.recv([t], src, 0))


def test_torchcomms_adapter_reconfigures_in_place():
    store = TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)
    addr = f"127.0.0.1:{store.port}"
    world = 2
    comms = [_LoopbackComm() for _ in range(world)]
    pgs = [ProcessGroupTorchComms(c, timeout=timedelta(seconds=20)) for c in comms]
    out = [None] * world
    errs = []

    def run(rank):
        try:
            pg = pgs[rank]
            for q in (1, 2):  # two quorums over the SAME communicator object
                pg.configure(f"{addr}/tc/{q}", f"r{rank}", rank, world, quorum_id=q)
                assert pg.size() == world
                t = torch.full((4,), float(rank + 1))
                pg.allreduce([t], dist.ReduceOp.SUM).wait()
                assert t.tolist() == [3.0] * 4
                b = torch.full((3,), float(rank))
                o = dist.BroadcastOptions()
                o.rootRank = 1
                w = pg.broadcast([b], o)
                w.wait()
                assert w.get_future().value() == [b] and b.tolist() == [1.0] * 3
                gathered = [torch.zeros(2) for _ in range(world)]
                pg.allgather([gathered], [torch.full((2,), float(rank))], None).wait()
                assert [g[0].item() for g in gathered] == [0.0, 1.0]
                if rank == 0:
                    pg.send([torch.arange(5.0)], 1, 0).wait()
                else:
                    r = torch.zeros(5)
                    pg.recv([r], 0, 0).wait()
                    assert r.tolist() == [0, 1, 2, 3, 4]
                pg.barrier().wait()
            out[rank] = comms[rank].reconfigures
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    [t.start() for t in ts]
    [t.join(60) for t in ts]
    assert not errs, errs
    assert out == [2, 2]
    assert pgs[0].getBackendName() == "torchcomms:loopback-gloo"
    with pytest.raises(ValueError):
        pgs[0].allreduce([torch.zeros(1), torch.zeros(1)], dist.ReduceOp.SUM)
    pgs[0].abort()
    assert comms[0].finalized
    with pytest.raises(RuntimeError):
        pgs[0].barrier()
    pgs[1].shutdown()


def test_torchx_component_spec_and_import_gate():
    from torchft_b200 import torchx as tx

    roles = tx.hsdp_spec("--lr", "1", replicas=3, workers_per_replica=2, script="train.py", gpus_per_node=8)
    assert [r.name for r in roles] == [f"replica_group_{i}" for i in range(3)]
    assert roles[2].env["REPLICA_GROUP_ID"] == "2" and roles[2].env["NUM_REPLICA_GROUPS"] == "3"
    assert "--master_port=29602" in roles[2].args and roles[2].args[-3:] == ["train.py", "--lr", "1"]
    assert roles[1].env["CUDA_VISIBLE_DEVICES"] == "2,3"
    try:
        import torchx  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError):
            tx.hsdp(replicas=2)


def test_torchx_component_builds_an_appdef_against_the_torchx_specs_api(monkeypatch):
    """torchx is not in this image: run the component against a stand-in ``torchx.specs`` with the real constructors'
    keyword names (specs.resource / Role / AppDef, reference torchft/torchx.py:60-89) so the conversion code executes."""
    import sys
    import types

    from torchft_b200 import torchx as tx

    specs = types.ModuleType("torchx.specs")

    class _Rec:
        def __init__(self, **kw):
            self.__dict__.update(kw)

    class Role(_Rec):
        pass

    class AppDef(_Rec):
        pass

    specs.Role, specs.AppDef = Role, AppDef
    specs.resource = lambda cpu, gpu, memMB, h=None: ("res", cpu, gpu, memMB, h)
    pkg = types.ModuleType("torchx")
    pkg.specs = specs
    monkeypatch.setitem(sys.modules, "torchx", pkg)
    monkeypatch.setitem(sys.modules, "torchx.specs", specs)
    monkeypatch.setenv("TORCHFT_LIGHTHOUSE", "http://lh:29510")
    app = tx.hsdp("--steps", "7", replicas=2, workers_per_replica=4, max_restarts=3, script="train.py", image="img:1",
                  env={"FOO": "bar"}, gpu=4, cpu=16, memMB=4096)
    assert isinstance(app, AppDef) and app.name == "torchft_b200" and len(app.roles) == 2
    r1 = app.roles[1]
    assert isinstance(r1, Role) and r1.name == "replica_group_1" and r1.image == "img:1" and r1.max_retries == 0  # restarts are torchrun's job
    assert r1.num_replicas == 1 and r1.min_replicas == 1 and r1.resource == ("res", 16, 4, 4096, None)
    assert r1.env["REPLICA_GROUP_ID"] == "1" and r1.env["NUM_REPLICA_GROUPS"] == "2" and r1.env["FOO"] == "bar"
    assert r1.env["TORCHFT_LIGHTHOUSE"] == "http://lh:29510"
    assert "--nproc_per_node=4" in " ".join(r1.args).replace("--nproc-per-node", "--nproc_per_node") and r1.args[-3:] == ["train.py", "--steps", "7"]
    assert "--master_port=29601" in r1.args and any(a.replace("-", "_") == "__max_restarts=3" for a in r1.args)


def test_failure_injector_comms_and_stall():
    pg = FakeProcessGroupWrapper(ProcessGroupDummy(0, 1))
    aborted = []
    pg.abort = lambda: aborted.append(True)  # type: ignore[method-assign]
    inj = FailureInjector(pg=pg).start()
    try:
        assert send_failure(inj.port, Failure.COMMS) == "ok"
        deadline = time.time() + 5
        while not aborted and time.time() < deadline:
            time.sleep(0.01)
        assert aborted
        assert send_failure(inj.port, Failure.STALL_PEER) == "ok"
        assert inj.stalled.wait(5)
        t = threading.Thread(target=inj.maybe_stall, daemon=True)
        t.start()
        t.join(0.2)
        assert t.is_alive()  # a stalled peer never proceeds
        inj.stalled.clear()
        t.join(2)
        assert not t.is_alive()
        # unknown commands are refused and do not kill the listener
        import socket

        with socket.create_connection(("127.0.0.1", inj.port), timeout=5) as s:
            s.sendall(b"bogus\n")
            assert b"unknown" in s.recv(64)
    finally:
        inj.stop()


@pytest.mark.parametrize("kind,check", [("kill_proc", lambda rc: rc == 1), ("segfault", lambda rc: rc < 0)])
def test_failure_injector_fatal_kinds(kind, check):
    code = (
        "import sys, time; sys.path.insert(0, %r)\n"
        "from torchft_b200.failure import FailureInjector\n"
        "inj = FailureInjector().start(); print(inj.port, flush=True); time.sleep(30)\n" % ROOT
    )
    p = subprocess.Popen([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    try:
        port = int(p.stdout.readline())
        send_failure(port, Failure(kind))
        rc = p.wait(20)
        assert check(rc), rc
    finally:
        if p.poll() is None:
            p.kill()


@pytest.mark.timeout(240)
def test_orchestrator_runs_groups_to_completion(tmp_path):
    env = dict(os.environ, USE_CPU="1", TRAIN_STEPS="12", CUDA_VISIBLE_DEVICES="")
    p = subprocess.run(
        [sys.executable, os.path.join(ROOT, "examples/orchestrator/train_orchestrated.py"), "--replicas", "2",
         "--min-replicas", "1", "--join-timeout-ms", "1000", "--log-dir", str(tmp_path), os.path.join(ROOT, "train_ddp.py")],
        env=env, capture_output=True, text=True, timeout=220)
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("finished") == 2, p.stdout
    logs = "".join(open(os.path.join(tmp_path, f)).read() for f in os.listdir(tmp_path) if f.endswith(".log"))
    assert '"final_step": 12' in logs


@pytest.mark.timeout(280)
def test_chaos_soak_ends_with_identical_weights(tmp_path):
    """Orchestrator + failure injection (kills from outside, in-process exit, comm aborts) over the CPU data plane:
    every group must finish at the target step with bit-identical weights."""
    import json

    out = tmp_path / "soak.json"
    env = dict(os.environ, USE_CPU="1", CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench/chaos_soak.py"), "--steps", "200", "--mtbf-secs", "5",
                        "--failures", "kill_proc,comms,kill_group", "--min-replicas", "2", "--max-failures", "1", "--timeout", "240", "--out", str(out)],
                       env=env, capture_output=True, text=True, timeout=270)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-2000:]
    res = json.loads(out.read_text())
    assert res["pass"] and res["final_weights_identical"] and res["n_injected"] >= 1, res


def test_slurm_runner_resubmits_only_dead_replica_groups(tmp_path):
    """examples/slurm/runner.py against fake sbatch/squeue: every replica group is submitted once, a group that
    disappears from the queue is re-submitted, live ones are left alone."""
    import stat
    import time

    state = tmp_path / "queue.txt"
    log = tmp_path / "sbatch.log"
    state.write_text("")
    (tmp_path / "sbatch").write_text(
        "#!/bin/bash\n"
        f"echo \"$@\" >> {log}\n"
        "name=$(printf '%s\\n' \"$@\" | sed -n 's/^--job-name=//p')\n"
        f"jid=$((1000 + $(wc -l < {log})))\n"
        f"echo \"$name $jid\" >> {state}\n"
        "echo $jid\n")
    (tmp_path / "squeue").write_text(f"#!/bin/bash\ncat {state}\n")
    for f in ("sbatch", "squeue"):
        os.chmod(tmp_path / f, os.stat(tmp_path / f).st_mode | stat.S_IEXEC)
    env = dict(os.environ, PATH=f"{tmp_path}:{os.environ['PATH']}")
    p = subprocess.Popen([sys.executable, os.path.join(ROOT, "examples/slurm/runner.py"), "--replicas", "3", "--check-every", "0.2",
                          "--job-name", "tft", "--script", "train.py", "--lighthouse", "http://lh:1"],
                         env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        deadline = time.time() + 20
        while len(state.read_text().splitlines()) < 3 and time.time() < deadline:
            time.sleep(0.05)
        time.sleep(0.6)  # a few more polls: nothing new may be submitted while all three are alive
        assert len(log.read_text().splitlines()) == 3
        first = log.read_text().splitlines()[1]
        assert "--job-name=tft_1" in first and "REPLICA_GROUP_ID=1,NUM_REPLICA_GROUPS=3,TORCHFT_LIGHTHOUSE=http://lh:1" in first
        assert "--master_port=29601 train.py" in first
        # replica group 1 dies (leaves the queue): only that one comes back. The queue is replaced atomically: a poll
        # between a truncate and the rewrite would see an empty queue and resubmit every group.
        (tmp_path / "queue.new").write_text("".join(l + "\n" for l in state.read_text().splitlines() if not l.startswith("tft_1 ")))
        os.replace(tmp_path / "queue.new", state)
        deadline = time.time() + 20
        while len(log.read_text().splitlines()) < 4 and time.time() < deadline:
            time.sleep(0.05)
        time.sleep(0.5)
        lines = log.read_text().splitlines()
        assert len(lines) == 4 and "--job-name=tft_1" in lines[3]
    finally:
        p.kill()
        p.wait()


def test_punisher_kills_a_replica_through_the_lighthouse(tmp_path):
    """examples/slurm/punisher.py kill_one -> Lighthouse /status.json -> POST /replica/<id>/kill -> ManagerServer.Kill RPC
    -> the victim process exits with code 1 (the reference's dashboard Kill button does the same)."""
    from datetime import timedelta

    from torchft_b200.bench_utils import loopback
    from torchft_b200.coordination import LighthouseServer

    lh = LighthouseServer(bind="[::]:0", min_replicas=1, join_timeout_ms=100, quorum_tick_ms=10)
    addr = loopback(lh.address())
    victim_code = (
        "import sys, time; sys.path.insert(0, %r)\n"
        "from datetime import timedelta\n"
        "from torchft_b200.coordination import ManagerServer, ManagerClient\n"
        "T = timedelta(seconds=10)\n"
        "ms = ManagerServer(replica_id='victim', lighthouse_addr=%r, hostname='127.0.0.1', bind='127.0.0.1:0', store_addr='s:1',\n"
        "                   world_size=1, heartbeat_interval=timedelta(milliseconds=50), connect_timeout=T, quorum_retries=0)\n"
        "ManagerClient(ms.address(), T)._quorum(0, 3, '', False, T, 0, True)\n"
        "print('joined', flush=True); time.sleep(60)\n" % (ROOT, addr))
    p = subprocess.Popen([sys.executable, "-c", victim_code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        assert p.stdout.readline().strip() == "joined"
        r = subprocess.run([sys.executable, os.path.join(ROOT, "examples/slurm/punisher.py"), "kill_one", "--lighthouse", addr],
                           capture_output=True, text=True, timeout=60)
        assert r.returncode == 0, r.stdout + r.stderr
        assert p.wait(20) == 1
    finally:
        if p.poll() is None:
            p.kill()
        lh.shutdown()


def test_launch_local_relaunches_failed_roles_until_they_succeed(tmp_path):
    """launcher.launch_local(relaunch=True): a role that exits non-zero is started again (poor man's scheduler)."""
    from torchft_b200.launcher import Role, launch_local

    marker = tmp_path / "attempts"
    script = tmp_path / "flaky.py"
    script.write_text(
        "import os, sys\n"
        f"p = {str(marker)!r}\n"
        "n = int(open(p).read()) if os.path.exists(p) else 0\n"
        "open(p, 'w').write(str(n + 1))\n"
        "sys.exit(0 if n >= 2 else 3)\n")
    ok = tmp_path / "ok.py"
    ok.write_text("print('fine')\n")
    roles = [Role(name="flaky", entrypoint=sys.executable, args=[str(script)]),
             Role(name="steady", entrypoint=sys.executable, args=[str(ok)], env={"X": "1"})]
    assert launch_local(roles, poll_s=0.1, relaunch=True) == 0
    assert marker.read_text() == "3"  # failed twice, succeeded on the third launch
    marker.unlink()
    assert launch_local(roles[:1], poll_s=0.1, relaunch=False) == 3  # without relaunch the exit code is reported
