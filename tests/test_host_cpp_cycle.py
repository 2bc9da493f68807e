"""The C++ host mirror's cycle shells (kube_batch_b200/host/kbhost.hpp, kb::actions::cycle: the twin of go/kbgpu/cycle.go)
against the oracle.

CPU: the flattened Running table (FlattenRunning, what kb_session_load_running receives) equals builder.py's
meta["running"] array for array, and the programs fail loudly without a device.  GPU (-m gpu): the reference's
preempt_test.go / reclaim_test.go restated in C++ (tests/host/evict_test.cpp), and random clusters run through
tests/host/cycle_run: one kb_cycle per session, replayed action by action through Session::Evict / Statement /
Session::Pipeline / Session::Allocate.  The binds the FakeBinder saw, the evictions the FakeEvictor saw (in call order),
every node's Idle / Releasing / Used (bit for bit) and every task's status must be what kbo.cycle computes on the same
objects.  The node state is what tests the replay's claims: reclaim's evictions replayed before its pipelines, preempt's
decisions in one Statement, each shell's slice taken from `bounds`."""
from __future__ import annotations

import os
import subprocess

import numpy as np
import pytest

from conftest import has_gpu
from kube_batch_b200 import abi, builder as B
from test_evict_parity import tier_variants

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "tests", "host")
ACTION_LISTS = (("reclaim", "allocate", "backfill", "preempt"), ("reclaim", "allocate"), ("allocate", "backfill", "preempt"))
STATUS = {"Pending": 1, "Allocated": 2, "Pipelined": 4, "Binding": 8, "Bound": 16, "Running": 32, "Releasing": 64, "Succeeded": 128}
READY = (STATUS["Allocated"], STATUS["Binding"], STATUS["Bound"], STATUS["Running"], STATUS["Succeeded"])   # ReadyTaskNum


def _build():
    if not os.path.exists(os.path.join(ROOT, "kube_batch_b200", "libkbgpu.so")):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "kube_batch_b200", "csrc")])
    subprocess.check_call(["make", "-C", HOST, "-f", "cycle.mk", "-s", "evict_test", "cycle_run"])


# ------------------------------------------------------------------------------------------------ clusters and their text form
def random_cluster(seed: int, big: bool = False) -> B.SessionBuilder:
    """Running, terminating and Pending pods of several PodGroups in several queues; some system-critical (kube-system or a
    critical priority class), some with scalars, some best-effort.  big: a few hundred nodes, filled, with hundreds of
    PodGroups waiting."""
    rng = np.random.default_rng(9100 + seed)
    b = B.SessionBuilder()
    nq = int(rng.integers(1, 4))
    for q in range(nq):
        b.add_queue(B.Queue(f"q{q}", int(rng.integers(1, 4)), creation=int(rng.integers(0, 3))))
    nn = int(rng.integers(2, 9)) if not big else int(rng.integers(150, 300))
    gpu_nodes = rng.random() < 0.4
    for n in range(nn):
        alloc = {"cpu": 8, "memory": 32e9, "pods": int(rng.integers(6, 14))}
        if gpu_nodes:
            alloc["nvidia.com/gpu"] = 4
        b.add_node(B.Node(f"n{n:04d}", alloc))
    cap = {f"n{n:04d}": 8.0 for n in range(nn)}
    k = 0
    for g in range(int(rng.integers(2, 9)) if not big else 3 * nn):
        ns = "kube-system" if rng.random() < 0.1 else "ns"
        b.add_pod_group(B.PodGroup(ns, f"g{g}", f"q{int(rng.integers(0, nq))}", min_member=int(rng.integers(0, 4)),
                                   priority=int(rng.integers(0, 3)), creation=int(rng.integers(0, 4))))
        cpu = float(rng.choice([0.5, 1, 2, 3]))
        req = {"cpu": cpu, "memory": cpu * 1e9}
        if gpu_nodes and rng.random() < 0.3:
            req["nvidia.com/gpu"] = 1
        best_effort = rng.random() < 0.1
        for i in range(int(rng.integers(1, 7))):
            state = rng.choice(["Running", "Running", "Pending", "Pending", "Deleting"])
            node = ""
            if state != "Pending":
                free = [n for n, c in cap.items() if c >= cpu]
                if not free:
                    state = "Pending"
                else:
                    node = str(rng.choice(free))
                    cap[node] -= cpu
            labels = {"priorityClassName": "system-node-critical"} if rng.random() < 0.05 else {}
            b.add_pod(B.Pod(ns, f"g{g}-p{i}", node, "Pending" if state == "Pending" else "Running",
                            {} if best_effort and state == "Pending" else dict(req), group=f"g{g}", labels=labels,
                            priority=int(rng.integers(0, 3)), creation=int(rng.integers(0, 5)) if rng.random() < 0.5 else k,
                            deleting=(state == "Deleting"), uid=f"{ns}-g{g}-p{i}"))
            k += 1
    return b


def _res(rl) -> str:
    return " ".join(f"{k}={float(v)!r}" for k, v in rl.items())


def _flag(v) -> int:
    return -1 if v is None else int(bool(v))


def write_cluster(path: str, b: B.SessionBuilder, cases=()):
    """The objects of `b` and the (label, actions, PluginConf) cases in cycle_run's input format."""
    lines = []
    for q in b.queues:
        lines.append(f"queue {q.name} {q.weight} {q.creation}")
    for n in b.nodes:
        assert not (n.labels or n.taints or n.unschedulable or n.ready is not None or n.network_unavailable is not None or
                    n.memory_pressure or n.disk_pressure or n.pid_pressure), "cycle_run carries no node labels, taints or conditions"
        lines.append(f"node {n.name} {_res(n.allocatable)}")
    for g in b.pod_groups:
        lines.append(f"podgroup {g.namespace} {g.name} {g.queue} {g.min_member} {g.priority} {g.creation}")
    for p in b.pods:
        assert not (p.init_requests or p.node_selector or p.affinity_terms or p.preferred_terms or p.tolerations or p.host_ports or
                    p.limits or p.pod_affinity or p.pod_anti_affinity), "cycle_run carries requests, priority and priority class only"
        assert set(p.labels) <= {"priorityClassName"}
        lines.append(f"pod {p.namespace} {p.name} {p.uid or p.namespace + '-' + p.name} {p.node_name or '-'} {p.phase} {int(p.deleting)} "
                     f"{1 if p.priority is None else p.priority} {p.creation} {p.group} {p.labels.get('priorityClassName', '-')} {_res(p.requests)}")
    for label, acts, conf in cases:
        lines.append(f"case {label} {','.join(acts)}")
        for tier in conf.tiers:
            lines.append("tier")
            for o in tier:
                flags = " ".join(str(_flag(getattr(o, f))) for f in (
                    "enabled_job_order", "enabled_job_ready", "enabled_job_pipelined", "enabled_task_order", "enabled_preemptable",
                    "enabled_reclaimable", "enabled_queue_order", "enabled_predicate", "enabled_node_order"))
                args = " ".join(f"{k}={v}" for k, v in o.arguments.items())
                lines.append(f"plugin {o.name} {flags} {args}".rstrip())
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")


def run_cases(tmp_path, b: B.SessionBuilder, cases):
    """cycle_run on `cases` -> {label: {"binds": {task: node}, "evicts": [task...], "nodes": {name: {what: {dim: v}}},
    "tasks": {task: status}}}"""
    path = str(tmp_path / "cluster.txt")
    write_cluster(path, b, cases)
    p = subprocess.run([os.path.join(HOST, "cycle_run"), path], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    out, cur = {}, None
    for line in p.stdout.splitlines():
        w = line.split()
        if w[0] == "case":
            cur = out[w[1]] = {"binds": {}, "evicts": [], "nodes": {}, "tasks": {}}
        elif w[0] == "bind":
            cur["binds"][w[1]] = w[2]
        elif w[0] == "evict":
            cur["evicts"].append(w[1])
        elif w[0] == "node":
            res, what = {}, None
            for tok in w[2:]:
                if "=" in tok:
                    k, v = tok.split("=")
                    res[what][k] = float(v)
                else:
                    what = tok
                    res[what] = {}
            cur["nodes"][w[1]] = res
        elif w[0] == "task":
            cur["tasks"][w[1]] = int(w[2])
        else:
            assert w[0] == "end", line
    return out


# ------------------------------------------------------------------------------------------------ the Running table (CPU)
def _running_table(tmp_path, b: B.SessionBuilder):
    path = str(tmp_path / "cluster.txt")
    write_cluster(path, b)
    p = subprocess.run([os.path.join(HOST, "cycle_run"), "--running", path], capture_output=True, text=True, check=True)
    dims, rows, waiting = None, {}, None
    for line in p.stdout.splitlines():
        w = line.split()
        if w[0] == "dims":
            dims = w[1:]
        elif w[0] == "running":
            rows[w[1]] = w[2:]
        else:
            assert w[0] == "waiting"
            waiting = [int(x) for x in w[1:]]
    return dims, rows, waiting


def check_running_table(tmp_path, b: B.SessionBuilder):
    """FlattenRunning == builder.flatten().meta["running"], array for array (rows matched by task name: the C++ table lists
    the tasks node by node, builder.py in object order; every array entry is per task)."""
    s = b.flatten()
    rt = s.meta["running"]
    dims, rows, waiting = _running_table(tmp_path, b)
    assert dims == s.meta["dims"]
    assert sorted(rows) == sorted(rt["names"])
    n, R = len(rt["names"]), s.R
    got = {k: np.zeros(n, dtype=rt[k].dtype) for k in ("node", "job", "res_present", "uid_rank", "flags", "prio", "ctime")}
    got["resreq"] = np.zeros((R, n))
    for i, name in enumerate(rt["names"]):
        r = rows[name]
        for k, v in zip(("node", "job", "res_present", "uid_rank", "flags", "prio", "ctime"), r[:7]):
            got[k][i] = int(v)
        got["resreq"][:, i] = [float(x) for x in r[7:]]
    for k, v in got.items():
        assert np.array_equal(v, rt[k]), (k, v.tolist(), rt[k].tolist())
    assert waiting == [0] * s.J                                       # no action has pipelined anything at session open
    return rt


def test_flatten_running_on_a_fixed_cluster(tmp_path):
    _build()
    G = 1e9
    b = B.SessionBuilder()
    b.add_node(B.Node("n0", {"cpu": 8, "memory": 32 * G, "pods": 10, "nvidia.com/gpu": 4}))
    b.add_node(B.Node("n1", {"cpu": 4, "memory": 16 * G, "pods": 10}))
    b.add_node(B.Node("n2", {"cpu": 2, "memory": 4 * G, "pods": 10, "example.com/fpga": 2}))
    b.add_queue(B.Queue("q1", 1))
    b.add_queue(B.Queue("q2", 2, creation=3))
    b.add_pod_group(B.PodGroup("ns", "pgA", "q1", 2, priority=3, creation=1))
    b.add_pod_group(B.PodGroup("kube-system", "sys", "q2", 1))
    b.add_pod_group(B.PodGroup("ns", "pgB", "q2", 1))
    b.add_pod_group(B.PodGroup("ns", "lost", "no-such-queue", 1))               # dropped by cache.Snapshot: its tasks are no candidates
    pods = [
        B.Pod("ns", "a0", "n0", "Running", {"cpu": 2, "memory": 4 * G, "nvidia.com/gpu": 2}, group="pgA", priority=5, creation=7, uid="u-a0"),
        B.Pod("ns", "a1", "n1", "Running", {"cpu": 1, "memory": 1 * G}, group="pgA", creation=2, uid="u-a1",
              labels={"priorityClassName": "system-cluster-critical"}),
        B.Pod("ns", "a2", "n1", "Running", {"cpu": 1, "memory": 1 * G}, group="pgA", deleting=True, uid="u-a2"),   # Releasing
        B.Pod("ns", "a3", "n0", "Pending", {"cpu": 1, "memory": 1 * G}, group="pgA", uid="u-a3"),                  # Bound
        B.Pod("ns", "a4", "", "Pending", {"cpu": 1, "memory": 1 * G}, group="pgA", uid="u-a4"),
        B.Pod("kube-system", "s0", "n2", "Running", {"cpu": 0.5, "memory": 1 * G, "example.com/fpga": 1}, group="sys", uid="u-s0"),
        B.Pod("ns", "b0", "n2", "Running", {"cpu": 3, "memory": 1 * G}, group="pgB", uid="u-b0"),                  # does not fit: off the node
        B.Pod("ns", "b1", "n0", "Running", {}, group="pgB", creation=9, uid="u-00b1", labels={"priorityClassName": "system-node-critical"}),
        B.Pod("ns", "b2", "n1", "Succeeded", {"cpu": 1, "memory": 1 * G}, group="pgB", uid="u-b2"),
        B.Pod("ns", "l0", "n1", "Running", {"cpu": 1, "memory": 1 * G}, group="lost", uid="u-l0"),
    ]
    for p in pods:
        b.add_pod(p)
    rt = check_running_table(tmp_path, b)
    assert sorted(rt["names"]) == ["kube-system/s0", "ns/a0", "ns/a1", "ns/b1"]
    crit = {name: int(f) for name, f in zip(rt["names"], rt["flags"])}
    assert crit == {"ns/a0": 0, "ns/a1": abi.KB_RUNNING_CRITICAL, "kube-system/s0": abi.KB_RUNNING_CRITICAL, "ns/b1": abi.KB_RUNNING_CRITICAL}


@pytest.mark.parametrize("seed", range(40))
def test_flatten_running_on_random_clusters(tmp_path, seed):
    _build()
    check_running_table(tmp_path, random_cluster(seed, big=(seed % 10 == 9)))


def test_host_programs_fail_loudly_without_gpu(tmp_path):
    _build()
    if has_gpu():
        pytest.skip("a GPU is present: covered by the gpu tests")
    p = subprocess.run([os.path.join(HOST, "evict_test")], capture_output=True, text=True)
    assert p.returncode == 3, (p.returncode, p.stderr)
    assert "no CPU fallback" in p.stderr and "KB_E_CUDA" in p.stderr
    path = str(tmp_path / "cluster.txt")
    write_cluster(path, random_cluster(0), [("default", ACTION_LISTS[0], next(tier_variants())[1])])
    p = subprocess.run([os.path.join(HOST, "cycle_run"), path], capture_output=True, text=True)
    assert p.returncode == 3, (p.returncode, p.stderr)
    assert "no CPU fallback" in p.stderr and "KB_E_CUDA" in p.stderr


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_reference_preempt_and_reclaim_tests_in_cpp():
    _build()
    p = subprocess.run([os.path.join(HOST, "evict_test")], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    ok = [line for line in p.stdout.splitlines() if line.startswith("ok   case")]
    assert [line.rsplit(": ", 1)[1] for line in ok] == ["1 eviction(s)", "2 eviction(s)", "1 eviction(s)"], p.stdout


def compare_with_oracle(b: B.SessionBuilder, got: dict, acts, conf, what: str) -> int:
    """One case of cycle_run against kbo.cycle on the same objects -> number of evictions."""
    from oracle import kbo
    s = b.flatten()
    rt = s.meta["running"]
    o, ev, order = kbo.cycle(s, conf, actions=acts, running=rt)
    d = o.decisions
    tasks, nodes, jobs = s.meta["tasks"], s.meta["nodes"], s.meta["jobs"]
    job_of = {f"{p.namespace}/{p.name}": f"{p.namespace}/{p.group}" for p in b.pods}
    # backfill's phantom tasks (Allocated on no node) are not replayed: the jobs that have one are left out of the bind, status
    # and ready-count checks (their gang may count the phantom); the node state is checked everywhere, phantoms take no node
    phantom_jobs = {job_of[tasks[t]] for t in np.nonzero((d["kind"] == abi.KB_KIND_ALLOCATED) & (d["node"] < 0))[0]}
    want_binds = {tasks[t]: nodes[d["node"][t]] for t in np.nonzero(d["dispatched"])[0] if job_of[tasks[t]] not in phantom_jobs}
    have_binds = {k: v for k, v in got["binds"].items() if job_of[k] not in phantom_jobs}
    assert have_binds == want_binds, f"{what}: binds"
    want_evicts = [rt["names"][i] for i in np.argsort(order, kind="stable") if ev[i]]
    assert got["evicts"] == want_evicts, f"{what}: evictions"
    dims = s.meta["dims"]
    for i, name in enumerate(nodes):
        for what_, arr in (("idle", o.node_idle), ("releasing", o.node_releasing), ("used", o.node_used)):
            have = np.array([got["nodes"][name][what_].get(k, 0.0) for k in dims])
            assert np.array_equal(have, arr[:, i]), f"{what}: node {name} {what_}: {have.tolist()} != {arr[:, i].tolist()}"
    # statuses: what the oracle's decisions and evictions mean for every task of the session
    want_status = {}
    for t, name in enumerate(tasks):
        k = int(d["kind"][t])
        want_status[name] = (STATUS["Pending"] if k in (abi.KB_KIND_NONE, abi.KB_KIND_SKIPPED) else STATUS["Pipelined"] if k == abi.KB_KIND_PIPELINED
                             else STATUS["Binding"] if d["dispatched"][t] else STATUS["Allocated"])
    for i, name in enumerate(rt["names"]):
        want_status[name] = STATUS["Releasing"] if ev[i] else STATUS["Running"]
    for name, st in want_status.items():
        if job_of[name] not in phantom_jobs:
            assert got["tasks"][name] == st, f"{what}: status of {name}: {got['tasks'][name]} != {st}"
    for j, job in enumerate(jobs):
        if job not in phantom_jobs:
            ready = sum(1 for name, st in got["tasks"].items() if job_of[name] == job and st in READY)
            assert ready == int(o.job_ready[j]), f"{what}: ready tasks of {job}: {ready} != {int(o.job_ready[j])}"
    return int(ev.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(40))
def test_cycle_replay_matches_the_oracle_on_the_gpu(tmp_path, seed):
    _build()
    b = random_cluster(seed)
    cases = [(f"{tname}:{i}", acts, conf) for tname, conf in tier_variants() for i, acts in enumerate(ACTION_LISTS)]
    got = run_cases(tmp_path, b, cases)
    assert sorted(got) == sorted(label for label, _, _ in cases)
    for label, acts, conf in cases:
        compare_with_oracle(b, got[label], acts, conf, f"seed {seed} {label} {acts}")


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_cycle_replay_matches_the_oracle_on_larger_clusters_on_the_gpu(tmp_path, seed):
    _build()
    b = random_cluster(100 + seed, big=True)
    cases = [(f"{tname}:{i}", acts, conf) for tname, conf in tier_variants() if tname in ("default", "one_tier_all")
             for i, acts in enumerate(ACTION_LISTS)]
    got = run_cases(tmp_path, b, cases)
    evictions = [compare_with_oracle(b, got[label], acts, conf, f"big seed {seed} {label} {acts}") for label, acts, conf in cases]
    assert sum(evictions) >= 100, evictions
