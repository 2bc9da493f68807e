"""Node affinity and inter-pod (anti)affinity through the C++ host mirror (kube_batch_b200/host/kbhost.hpp: Flatten's
selector atoms, FlattenPodAffinity, FlattenRunning's group lists) — the twin of go/kbgpu/flatten.go and podaffinity.go.

CPU: tests/host/affinity_run --flat flattens the same objects builder.py flattens, and the tables are compared through
identities that do not depend on numbering (both flatteners number types, groups, kinds and key sets in an order of their own):
  * a key set is identified by the domain partition it gives the nodes (node_domain row);
  * a group by its key set plus the names of its members: the Running pods that list it in their group lists and the pending
    tasks that contribute to it;
  * a kind by its unbound flag plus the weight entries (task, key set, value) that name it.
Through them: the key sets, each group's counter per node and its total, per task forbid / need / contrib / self-match and
weight entries, kind counts per node, per Running pod KB_RUNNING_AFF_MEMBER and its groups.  Node affinity is compared as
relations: per (task, node) the required terms match and the preferred count.  Every cluster is flattened a second time from a
file that declares its nodes and pods in shuffled order: the output must be the same.  The limits throw, naming the limit.

GPU (-m gpu): the same objects through the Cycle shells and the per-action allocate / backfill shells against the oracle: binds,
evictions in order, node Idle / Releasing / Used bit for bit, task statuses."""
from __future__ import annotations

import collections
import json
import os
import subprocess

import numpy as np
import pytest

import aff_gen
import aff_gen_many
from conftest import has_gpu
from kube_batch_b200 import abi, builder as B
from kube_batch_b200.snapshot import PluginConf
from test_evict_parity import tier_variants
from test_host_cpp_cycle import compare_with_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "tests", "host")
PROG = os.path.join(HOST, "affinity_run")


def _build():
    if not os.path.exists(os.path.join(ROOT, "kube_batch_b200", "libkbgpu.so")):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "kube_batch_b200", "csrc")])
    subprocess.check_call(["make", "-C", HOST, "-f", "affinity.mk", "-s", "affinity_run"])


def builder_of(gen, *args, **kw) -> B.SessionBuilder:
    """The SessionBuilder of a generator that returns builder.flatten()"""
    flatten = B.SessionBuilder.flatten
    B.SessionBuilder.flatten = lambda self, W=1: self
    try:
        return gen(*args, **kw)
    finally:
        B.SessionBuilder.flatten = flatten


# ------------------------------------------------------------------------------------------------ the text form
def _res(rl) -> str:
    return " ".join(f"{k}={float(v)!r}" for k, v in rl.items())


def _vals(v) -> str:
    assert all(x and "," not in x and " " not in x for x in v)
    return ",".join(v) if v else "-"


def _s(x: str) -> str:
    assert " " not in x
    return x if x else "-"


def _flag(v) -> int:
    return -1 if v is None else int(bool(v))


def _pod_terms(kind: str, a: B.PodAffinity):
    out = [f"podaff {kind}"]
    for w, t in [("req", t) for t in a.required] + [(str(w), t) for (w, t) in a.preferred]:
        out.append(f"podterm {kind} {w} {_s(t.topology_key)} {_vals(t.namespaces)} {'nil' if t.nil_selector else 'sel'}")
        if not t.nil_selector:
            out += [f"matchlabel {k} {_s(v)}" for k, v in t.match_labels.items()]
            out += [f"matchexpr {k} {op} {_vals(list(vals))}" for (k, op, vals) in t.match_expressions]
    return out


def cluster_lines(b: B.SessionBuilder, cases=(), allocate=(), order=None):
    """The objects of `b` in affinity_run's input format.  allocate: (ns, name, node) placed by ssn.Allocate after the session
    opens.  order: a numpy Generator that shuffles the nodes and pods."""
    nodes, pods = list(b.nodes), list(b.pods)
    if order is not None:
        nodes = [nodes[i] for i in order.permutation(len(nodes))]
        pods = [pods[i] for i in order.permutation(len(pods))]
    lines = [f"queue {q.name} {q.weight} {q.creation}" for q in b.queues]
    for n in nodes:
        assert not (n.unschedulable or n.ready is not None or n.network_unavailable is not None or n.memory_pressure or
                    n.disk_pressure or n.pid_pressure), "affinity_run carries no node conditions"
        lines.append(f"node {n.name} {_res(n.allocatable)}")
        lines += [f"label {k} {_s(v)}" for k, v in n.labels.items()]
        lines += [f"taint {k} {_s(v)} {e}" for (k, v, e) in n.taints]
    lines += [f"podgroup {g.namespace} {g.name} {g.queue} {g.min_member} {g.priority} {g.creation}" for g in b.pod_groups]
    for p in pods:
        assert not (p.init_requests or p.limits), "affinity_run carries no init containers or limits"
        lines.append(f"pod {p.namespace} {p.name} {p.uid or p.namespace + '-' + p.name} {p.node_name or '-'} {p.phase} {int(p.deleting)} "
                     f"{1 if p.priority is None else p.priority} {p.creation} {p.group} {p.labels.get('priorityClassName', '-')} {_res(p.requests)}")
        lines += [f"label {k} {_s(v)}" for k, v in p.labels.items()]
        lines += [f"selector {k} {_s(v)}" for k, v in p.node_selector.items()]
        lines += [f"toleration {_s(k)} {_s(op)} {_s(v)} {_s(e)}" for (k, op, v, e) in p.tolerations]
        lines += [f"hostport {_s(ip)} {_s(proto)} {port}" for (ip, proto, port) in p.host_ports]
        if p.affinity_terms is not None:
            lines.append("required")
            for term in p.affinity_terms:
                lines.append("term")
                for (k, op, vals) in term:
                    lines.append(f"field {k[len('field:'):]} {op} {_vals(list(vals))}" if k.startswith("field:") else f"expr {k} {op} {_vals(list(vals))}")
        for (w, exprs) in p.preferred_terms:
            lines.append(f"preferred {w}")
            lines += [f"expr {k} {op} {_vals(list(vals))}" for (k, op, vals) in exprs]
        if p.pod_affinity is not None:
            lines += _pod_terms("aff", p.pod_affinity)
        if p.pod_anti_affinity is not None:
            lines += _pod_terms("anti", p.pod_anti_affinity)
    lines += [f"allocate {ns} {name} {node}" for (ns, name, node) in allocate]
    for label, acts, mode, conf in cases:
        lines.append(f"case {label} {','.join(acts)} {mode}")
        for tier in conf.tiers:
            lines.append("tier")
            for o in tier:
                flags = " ".join(str(_flag(getattr(o, f))) for f in (
                    "enabled_job_order", "enabled_job_ready", "enabled_job_pipelined", "enabled_task_order", "enabled_preemptable",
                    "enabled_reclaimable", "enabled_queue_order", "enabled_predicate", "enabled_node_order"))
                args = " ".join(f"{k}={v}" for k, v in o.arguments.items())
                lines.append(f"plugin {o.name} {flags} {args}".rstrip())
    return "\n".join(lines) + "\n"


def run_prog(tmp_path, text: str, *args):
    path = str(tmp_path / "cluster.txt")
    with open(path, "w") as f:
        f.write(text)
    return subprocess.run([PROG, *args, path], capture_output=True, text=True)


def flat(tmp_path, b: B.SessionBuilder, **kw) -> dict:
    p = run_prog(tmp_path, cluster_lines(b, **kw), "--flat")
    assert p.returncode == 0, p.stderr[-2000:]
    return json.loads(p.stdout)


# ------------------------------------------------------------------------------------------------ numbering-free views
def _relations(s, T, N):
    """(aff_match[T][N], pref_count[T][N]) from builder.py's arrays"""
    W = s.W
    labels = s.node_labels
    aff = np.ones((T, N), dtype=np.int64)
    pref = np.zeros((T, N), dtype=np.int64)
    for t in range(T):
        for n in range(N):
            k = int(s.task_n_aff_terms[t])
            if k:
                aff[t, n] = int(any(all((int(labels[w, n]) & int(s.task_aff_terms[i, w, t])) == int(s.task_aff_terms[i, w, t]) for w in range(W))
                                    for i in range(k)))
            for i in range(int(s.task_n_pref_terms[t])):
                if all((int(labels[w, n]) & int(s.task_pref_terms[i, w, t])) == int(s.task_pref_terms[i, w, t]) for w in range(W)):
                    pref[t, n] += int(s.task_pref_weights[i, t])
    return aff, pref


def view(pa: dict, tasks, running, run_groups, N, ignore_unbound=False):
    """kb_pod_affinity (as dict of arrays) -> its numbering-free content"""
    if pa is None:
        return None
    T = len(tasks)
    nks, ng, nk = int(pa["n_keysets"]), int(pa["n_groups"]), int(pa["n_kinds"])
    dom = np.asarray(pa["node_domain"], dtype=np.int64).reshape(-1)[: nks * N].reshape(nks, N)
    ks_id = [tuple(int(x) for x in dom[k]) for k in range(nks)]
    forbid = [set() for _ in range(T)]
    contrib = [set() for _ in range(T)]
    for t in range(T):
        f, c = int(pa["task_forbid"][t]), int(pa["task_contrib"][t])
        for g in range(min(ng, 64)):
            if (f >> g) & 1:
                forbid[t].add(g)
            if (c >> g) & 1:
                contrib[t].add(g)
        if ng > 64:
            off = pa["task_xgroup_off"]
            for e in np.asarray(pa["task_xgroup"]).reshape(-1)[int(off[t]): int(off[t + 1])]:
                e = int(e)
                if e & abi.KB_XGROUP_FORBID:
                    forbid[t].add(e >> 2)
                if e & abi.KB_XGROUP_CONTRIB:
                    contrib[t].add(e >> 2)
    members = [set() for _ in range(ng)]
    for name, gs in zip(running, run_groups):
        for g in gs:
            members[g].add(name)
    for t in range(T):
        for g in contrib[t]:
            members[g].add(tasks[t])
    gkeys = [int(x) for x in np.asarray(pa["group_keyset"]).reshape(-1)[:ng]]
    gid = [(ks_id[gkeys[g]], frozenset(members[g])) for g in range(ng)]
    count0 = np.asarray(pa["group_count0"]).reshape(-1)
    total0 = np.asarray(pa["group_total0"]).reshape(-1)
    kd = np.asarray(pa["keyset_domains"]).reshape(-1)
    groups, off = {}, 0
    for g in range(ng):
        row = dom[gkeys[g]]
        per_node = tuple(int(count0[off + row[n]]) if row[n] >= 0 else None for n in range(N))
        val = (per_node, int(total0[g]))
        assert groups.setdefault(gid[g], val) == val
        off += int(kd[gkeys[g]])
    woff = np.asarray(pa["task_weight_off"]).reshape(-1)
    wk, wks, wv = (np.asarray(pa[k]).reshape(-1) for k in ("weight_kind", "weight_keyset", "weight_value"))
    entries = collections.defaultdict(set)
    for t in range(T):
        for i in range(int(woff[t]), int(woff[t + 1])):
            entries[int(wk[i])].add((tasks[t], ks_id[int(wks[i])], int(wv[i])))
    ku = np.asarray(pa["kind_unbound"]).reshape(-1)
    kid = [(0 if ignore_unbound else int(ku[k]), frozenset(entries[k])) for k in range(nk)]
    kc = np.asarray(pa["node_kind_count0"], dtype=np.int64).reshape(-1)
    node_kinds = [collections.Counter() for _ in range(N)]
    for k in range(nk):
        for n in range(N):
            if kc[k * N + n]:
                node_kinds[n][kid[k]] += int(kc[k * N + n])
    task_kind = {tasks[t]: (kid[int(pa["task_kind"][t])] if int(pa["task_kind"][t]) >= 0 else None) for t in range(T)}
    per_task = {tasks[t]: (frozenset(gid[g] for g in forbid[t]), gid[int(pa["task_need"][t])] if int(pa["task_need"][t]) >= 0 else None,
                           frozenset(gid[g] for g in contrib[t]),
                           frozenset((kid[int(wk[i])], ks_id[int(wks[i])], int(wv[i])) for i in range(int(woff[t]), int(woff[t + 1]))))
                for t in range(T)}
    run = {name: frozenset(gid[g] for g in gs) for name, gs in zip(running, run_groups)}
    return {"keysets": set(ks_id), "groups": groups, "tasks": per_task, "task_kind": task_kind, "node_kinds": node_kinds, "running": run}


def cpp_view(got: dict, ignore_unbound=False):
    off, grp = got["running_aff_group_off"], got["running_aff_group"]
    rg = [grp[off[i]: off[i + 1]] for i in range(len(got["running"]))]
    pa = got["pod_affinity"]
    if pa is not None:
        pa = dict(pa)
        for k in ("task_forbid", "task_contrib"):
            pa[k] = [int(x) for x in pa[k]]
    return view(pa, got["tasks"], got["running"], rg, len(got["nodes"]), ignore_unbound)


def builder_view(s, ignore_unbound=False):
    rt, rag = s.meta["running"], s.meta["running_aff_groups"]
    off, grp = rag["aff_group_off"], rag["aff_group"]
    rg = [[int(g) for g in grp[off[i]: off[i + 1]]] for i in range(len(rt["names"]))]
    return view(s.pod_affinity, s.meta["tasks"], rt["names"], rg, len(s.meta["nodes"]), ignore_unbound)


def check_flat(tmp_path, b: B.SessionBuilder, seed=0, allocate=(), ignore_unbound=False):
    """affinity_run --flat against builder.flatten() on the same objects; returns the C++ output"""
    s = b.flatten()
    got = flat(tmp_path, b, allocate=allocate)
    assert got == flat(tmp_path, b, allocate=allocate, order=np.random.default_rng(seed)), "the declaration order changed the flattening"
    tasks, nodes = s.meta["tasks"], s.meta["nodes"]
    assert got["nodes"] == nodes and sorted(got["tasks"]) == sorted(tasks)
    ti = [got["tasks"].index(t) for t in tasks]
    T, N = len(tasks), len(nodes)
    aff, pref = _relations(s, T, N)
    assert np.array_equal(np.asarray(got["aff_match"]).reshape(-1, N)[ti] if T else aff, aff), "required node affinity"
    assert np.array_equal(np.asarray(got["pref_count"]).reshape(-1, N)[ti] if T else pref, pref), "preferred node affinity counts"
    assert [got["task_flags"][i] for i in ti] == [int(x) for x in s.task_flags[:T]], "task flags"
    assert got["flags"] == int(getattr(s, "flags", 0)), "snapshot flags"
    rt = s.meta["running"]
    assert sorted(got["running"]) == sorted(rt["names"])
    ri = {name: i for i, name in enumerate(got["running"])}
    assert [got["running_flags"][ri[name]] for name in rt["names"]] == [int(x) for x in rt["flags"]], "Running flags"
    if s.pod_affinity is None:
        assert got["pod_affinity"] is None
        return got
    assert got["pod_affinity"] is not None
    want, have = builder_view(s, ignore_unbound), cpp_view(got, ignore_unbound)
    for k in ("keysets", "groups", "tasks", "task_kind", "node_kinds", "running"):
        assert have[k] == want[k], k
    if not allocate:
        assert got["pod_affinity"]["first_unbound_node"] == -1
    return got


# ------------------------------------------------------------------------------------------------ CPU
G = 1e9
HOSTNAME, ZONE = aff_gen.HOST, aff_gen.ZONE


def fixed_cluster(unbound_on_node: bool):
    """Every branch of both flatteners: a nil selector, the default namespace, a pod matching its own required affinity, a needed
    group, Gt / Lt on a label that is not an integer, MatchFields on metadata.name, a preferred term with an empty topology key,
    taints, tolerations, host ports, a nodeSelector.  unbound_on_node: pod web-x is declared Pending (placed later by
    ssn.Allocate, so its Spec.NodeName stays ""), else Bound on n1."""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    for i, (zone, size) in enumerate([("a", "8"), ("a", "big"), ("b", "16"), ("c", "4")]):
        labels = {HOSTNAME: f"n{i}", ZONE: zone, "size": size}
        if i == 3:
            del labels[ZONE]
        n = B.Node(f"n{i}", {"cpu": 16, "memory": 64 * G, "pods": 20}, labels=labels)
        if i == 2:
            n.taints = [("dedicated", "gpu", "NoSchedule"), ("soft", "x", "PreferNoSchedule")]
        b.add_node(n)
    for g in ("run", "web", "db", "gt"):
        b.add_pod_group(B.PodGroup("default" if g == "db" else "ns", g, "q", 1))
    web = lambda: B.PodAffinity(required=[B.PodAffinityTerm(ZONE, match_labels={"app": "web"})])
    b.add_pod(B.Pod("ns", "run-0", "n0", "Running", {"cpu": 1, "memory": G}, group="run", labels={"app": "web"}, uid="u-r0",
                    pod_anti_affinity=B.PodAffinity(required=[B.PodAffinityTerm(HOSTNAME, match_labels={"app": "db"}, namespaces=["default"])])))
    b.add_pod(B.Pod("ns", "run-1", "n2", "Running", {"cpu": 1, "memory": G}, group="run", labels={"app": "db", "tier": "x"}, uid="u-r1",
                    host_ports=[("", "TCP", 8080)],
                    pod_affinity=B.PodAffinity(preferred=[(7, B.PodAffinityTerm(ZONE, match_labels={"app": "web"})),
                                                          (3, B.PodAffinityTerm("", match_labels={"app": "web"}))])))
    b.add_pod(B.Pod("ns", "web-x", "" if unbound_on_node else "n1", "Pending", {"cpu": 1, "memory": G}, group="run", labels={"app": "web"},
                    uid="u-wx", pod_affinity=B.PodAffinity(preferred=[(5, B.PodAffinityTerm(ZONE, match_labels={"app": "web"}))])))
    for i in range(2):      # needs a group of its own app: matches its own terms (self-match)
        b.add_pod(B.Pod("ns", f"web-{i}", "", "Pending", {"cpu": 1, "memory": G}, group="web", labels={"app": "web"}, uid=f"u-w{i}",
                        pod_affinity=web(), host_ports=[("", "TCP", 8080)], tolerations=[("dedicated", "Equal", "gpu", "NoSchedule")]))
    b.add_pod(B.Pod("default", "db-0", "", "Pending", {"cpu": 1, "memory": G}, group="db", labels={"app": "db"}, uid="u-d0",
                    node_selector={ZONE: "a"},
                    pod_affinity=B.PodAffinity(required=[B.PodAffinityTerm(HOSTNAME, nil_selector=True)]),
                    pod_anti_affinity=B.PodAffinity(preferred=[(2, B.PodAffinityTerm(HOSTNAME, match_expressions=[("tier", "Exists", [])]))])))
    b.add_pod(B.Pod("ns", "gt-0", "", "Pending", {"cpu": 1, "memory": G}, group="gt", uid="u-g0",
                    affinity_terms=[[("size", "Gt", ["6"])], [("size", "Lt", ["5"]), ("field:metadata.name", "In", ["n3"])]],
                    preferred_terms=[(10, [("size", "Gt", ["10"])]), (0, [(ZONE, "In", ["a"])]), (4, [(ZONE, "NotIn", ["a"])])]))
    b.add_pod(B.Pod("ns", "gt-1", "", "Pending", {}, group="gt", uid="u-g1",
                    affinity_terms=[[("field:metadata.name", "NotIn", ["n0"]), (ZONE, "Exists", [])]]))
    return b


def _builder_form(b: B.SessionBuilder) -> B.SessionBuilder:
    """builder.py has no MatchFields: its twin of the fixed cluster evaluates `metadata.name` as a node label of that name, and
    skips weight-0 preferred terms like the flatteners do"""
    import copy
    b2 = copy.deepcopy(b)
    for n in b2.nodes:
        n.labels["metadata.name"] = n.name
    for p in b2.pods:
        if p.affinity_terms:
            p.affinity_terms = [[(k[len("field:"):] if k.startswith("field:") else k, op, v) for (k, op, v) in term] for term in p.affinity_terms]
        p.preferred_terms = [(w, e) for (w, e) in p.preferred_terms if w]
    return b2


def test_fixed_cluster_flattens_like_builder(tmp_path):
    _build()
    b = fixed_cluster(unbound_on_node=False)
    s = _builder_form(b).flatten()
    got = flat(tmp_path, b)
    # the builder twin carries one more label per node: compare the relations, not the atoms
    tasks, N = s.meta["tasks"], len(s.meta["nodes"])
    ti = [got["tasks"].index(t) for t in tasks]
    aff, pref = _relations(s, len(tasks), N)
    assert np.array_equal(np.asarray(got["aff_match"])[ti], aff) and np.array_equal(np.asarray(got["pref_count"])[ti], pref)
    gt0 = got["tasks"].index("ns/gt-0")
    assert got["aff_match"][gt0] == [1, 0, 1, 1]          # size=big does not parse: Gt fails on n1; n3 by size < 5 and its name
    assert got["pref_count"][gt0] == [0, 0, 14, 4]        # n3 has no zone label: NotIn holds
    assert got["aff_match"][got["tasks"].index("ns/gt-1")] == [0, 1, 1, 0]
    want, have = builder_view(s), cpp_view(got)
    for k in ("keysets", "groups", "tasks", "task_kind", "node_kinds", "running"):
        assert have[k] == want[k], k
    fl = dict(zip(got["tasks"], got["task_flags"]))
    assert fl["ns/web-0"] & abi.KB_TASK_AFF_SELF_MATCH and not fl["default/db-0"] & abi.KB_TASK_AFF_SELF_MATCH
    assert fl["ns/gt-0"] & abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY and not fl["ns/gt-0"] & abi.KB_TASK_HAS_POD_AFFINITY
    assert got["flags"] == abi.KB_SNAPSHOT_PLACED_POD_AFFINITY
    pa = got["pod_affinity"]
    assert pa["task_need"][got["tasks"].index("ns/web-0")] >= 0 and pa["task_need"][got["tasks"].index("default/db-0")] >= 0
    assert got["running_flags"][got["running"].index("ns/run-0")] & abi.KB_RUNNING_AFF_MEMBER


def test_an_unbound_pod_on_a_node(tmp_path):
    """A task Allocated earlier in the session sits on its node with an empty Spec.NodeName: first_unbound_node is that node and
    its kind is unbound; everything else is what builder.py computes for the same pod bound there."""
    _build()
    got = flat(tmp_path, fixed_cluster(unbound_on_node=True), allocate=[("ns", "web-x", "n1")])
    pa = got["pod_affinity"]
    assert pa["first_unbound_node"] == 1
    N = len(got["nodes"])
    unbound_on = [sum(pa["node_kind_count0"][k * N + n] for k in range(pa["n_kinds"]) if pa["kind_unbound"][k]) for n in range(N)]
    assert unbound_on == [0, 1, 0, 0]
    s = _builder_form(fixed_cluster(unbound_on_node=False)).flatten()
    want, have = builder_view(s, ignore_unbound=True), cpp_view(got, ignore_unbound=True)
    for k in ("keysets", "groups", "tasks", "node_kinds", "running"):
        assert have[k] == want[k], k


@pytest.mark.parametrize("seed", range(40))
def test_random_affinity_sessions_flatten_like_builder(tmp_path, seed):
    _build()
    check_flat(tmp_path, aff_gen.random_affinity_session(seed, node_pref=seed % 2 == 1, besteffort=seed % 4 == 2), seed)


@pytest.mark.parametrize("seed", range(10))
def test_sessions_with_more_than_64_groups_flatten_like_builder(tmp_path, seed):
    _build()
    b = aff_gen_many.random_affinity_session(50 + seed, n_nodes=10 + seed, n_groups=120, n_apps=48)
    got = check_flat(tmp_path, b, seed)
    assert got["pod_affinity"]["n_groups"] > 64 and "task_xgroup_off" in got["pod_affinity"]


@pytest.mark.parametrize("seed", range(6))
def test_host_spread_and_evict_spread_clusters_flatten_like_builder(tmp_path, seed):
    _build()
    check_flat(tmp_path, aff_gen.host_spread_session(seed, ports=seed % 2 == 1), seed)
    got = check_flat(tmp_path, builder_of(aff_gen.evict_spread_cluster, seed, members_running=True), seed)
    if got["pod_affinity"] is not None:
        assert all(bool(f & abi.KB_RUNNING_AFF_MEMBER) == (got["running_aff_group_off"][i + 1] > got["running_aff_group_off"][i])
                   for i, f in enumerate(got["running_flags"]))


def test_sessions_without_terms_keep_their_atoms(tmp_path):
    _build()
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_node(B.Node("n0", {"cpu": 4, "memory": 8 * G, "pods": 10}, labels={"disk": "ssd"}))
    b.add_pod_group(B.PodGroup("ns", "g", "q", 1))
    b.add_pod(B.Pod("ns", "p", "", "Pending", {"cpu": 1, "memory": G}, group="g", node_selector={"disk": "ssd"}, uid="u-p"))
    got = check_flat(tmp_path, b)
    assert got["pod_affinity"] is None and got["flags"] == 0 and got["task_n_pref"] == [0] and got["running_aff_group_off"] == [0]


def test_a_preferred_term_without_expressions_matches_no_node(tmp_path):
    """NodeSelectorRequirementsAsSelector of an empty list is labels.Nothing() (helpers.go:205-208): the term adds its weight
    nowhere (builder.py lets such a term match every node)"""
    _build()
    got = flat(tmp_path, _one_pod_session(preferred_terms=[(5, []), (3, [(HOSTNAME, "Exists", [])])]))
    assert got["pref_count"] == [[3]] and got["task_n_pref"] == [2]


# ---- refusals: every limit throws and names itself
def _one_pod_session(**kw):
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_node(B.Node("n0", {"cpu": 4, "memory": 8 * G, "pods": 10}, labels={HOSTNAME: "n0"}))
    b.add_pod_group(B.PodGroup("ns", "g", "q", 1))
    b.add_pod(B.Pod("ns", "p", "", "Pending", {"cpu": 1, "memory": G}, group="g", uid="u-p", **kw))
    return b


def _refused(tmp_path, b, what):
    p = run_prog(tmp_path, cluster_lines(b), "--flat")
    assert p.returncode == 1 and "unsupported session" in p.stderr and what in p.stderr, p.stderr


def test_refusals_name_the_limit(tmp_path):
    _build()
    _refused(tmp_path, _one_pod_session(affinity_terms=[[("k", "In", [str(i)])] for i in range(abi.KB_MAX_AFF_TERMS + 1)]), "KB_MAX_AFF_TERMS")
    _refused(tmp_path, _one_pod_session(preferred_terms=[(1, [("k", "In", [str(i)])]) for i in range(abi.KB_MAX_PREF_TERMS + 1)]), "KB_MAX_PREF_TERMS")
    _refused(tmp_path, _one_pod_session(affinity_terms=[[("k", "NotIn", [str(i)]) for i in range(64 * abi.KB_MAX_W + 1)]]), "KB_MAX_W")
    _refused(tmp_path, _one_pod_session(pod_affinity=B.PodAffinity(required=[B.PodAffinityTerm("", match_labels={"a": "b"})])), "empty topologyKey")
    b = _one_pod_session()
    b.pods.clear()
    for i in range(65):     # 65 key sets, one group each
        b.add_pod(B.Pod("ns", f"k{i}", "", "Pending", {"cpu": 1, "memory": G}, group="g", uid=f"u-k{i}",
                        pod_anti_affinity=B.PodAffinity(required=[B.PodAffinityTerm(f"key{i}", match_labels={"a": "b"})])))
    _refused(tmp_path, b, "topology key sets: more than 64")
    b.pods.clear()
    for i in range(4097):   # 4097 groups on one key set
        b.add_pod(B.Pod("ns", f"g{i}", "", "Pending", {"cpu": 1, "memory": G}, group="g", uid=f"u-g{i}",
                        pod_anti_affinity=B.PodAffinity(required=[B.PodAffinityTerm(HOSTNAME, match_labels={"app": str(i)})])))
    _refused(tmp_path, b, "KB_MAX_AFF_GROUPS")


def test_affinity_run_fails_loudly_without_gpu(tmp_path):
    _build()
    if has_gpu():
        pytest.skip("a GPU is present: covered by the gpu tests")
    p = run_prog(tmp_path, cluster_lines(aff_gen.random_affinity_session(0), [("c", ("allocate", "backfill"), "cycle", PluginConf.default())]))
    assert p.returncode == 3 and "no CPU fallback" in p.stderr and "KB_E_CUDA" in p.stderr, (p.returncode, p.stderr)


# ------------------------------------------------------------------------------------------------ GPU
def run_cases(tmp_path, b, cases):
    p = run_prog(tmp_path, cluster_lines(b, cases))
    out, cur = {}, None
    for line in p.stdout.splitlines():
        w = line.split()
        if w[0] == "case":
            cur = out[w[1]] = {"binds": {}, "evicts": [], "nodes": {}, "tasks": {}, "error": None}
        elif w[0] == "error":
            cur["error"] = line
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
    assert p.returncode in (0, 1), p.stderr[-2000:]
    return out


def _check_cases(tmp_path, b, cases, what, follow=False):
    got = run_cases(tmp_path, b, cases)
    assert sorted(got) == sorted(c[0] for c in cases), what
    for label, acts, _, conf in cases:
        assert got[label]["error"] is None, f"{what} {label}: {got[label]['error']}"
        if follow:
            import follow_oracle
            from oracle import kbo
            saved = kbo.cycle

            def followed(*a, **kw):       # follow_oracle.cycle calls kbo.cycle itself
                kbo.cycle = saved
                try:
                    return follow_oracle.cycle(*a, **kw)
                finally:
                    kbo.cycle = followed
            kbo.cycle = followed
            try:
                compare_with_oracle(b, got[label], acts, conf, f"{what} {label}")
            finally:
                kbo.cycle = saved
        else:
            compare_with_oracle(b, got[label], acts, conf, f"{what} {label}")


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(12))
def test_random_affinity_sessions_through_the_shells_on_the_gpu(tmp_path, seed):
    _build()
    b = aff_gen.random_affinity_session(seed, node_pref=seed % 2 == 1, besteffort=seed % 3 == 0)
    cases = [(f"{tname}:{mode}", ("allocate", "backfill"), mode, conf) for tname, conf in tier_variants() for mode in ("cycle", "shells")]
    _check_cases(tmp_path, b, cases, f"seed {seed}")


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(4))
def test_preferred_zone_terms_on_and_off_the_pipeline_on_the_gpu(tmp_path, seed):
    _build()
    for p_affine in (0.0, 0.6):         # without inter-pod terms the session runs on the pipeline, with them on the per-visit kernels
        b = aff_gen.random_affinity_session(300 + seed, node_pref=True, p_affine=p_affine)
        cases = [(f"{tname}", ("allocate", "backfill"), "cycle", conf) for tname, conf in tier_variants() if tname in ("default", "one_tier_all")]
        _check_cases(tmp_path, b, cases, f"seed {seed} p_affine {p_affine}")


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(8))
def test_evicting_actions_with_members_and_soft_affinity_on_the_gpu(tmp_path, seed):
    _build()
    from test_evict_pod_pref import pod_pref_cluster
    acts = ("reclaim", "allocate", "backfill", "preempt")
    confs = [(t, c) for t, c in tier_variants() if t in ("default", "one_tier_all", "drf_first")]
    b = builder_of(aff_gen.evict_spread_cluster, seed, members_running=True)
    _check_cases(tmp_path, b, [(t, acts, "cycle", c) for t, c in confs], f"spread seed {seed}", follow=True)
    b = builder_of(pod_pref_cluster, seed)
    _check_cases(tmp_path, b, [(t, acts, "cycle", c) for t, c in confs], f"soft seed {seed}", follow=True)


@pytest.mark.gpu
def test_a_class_that_reads_a_counter_group_refuses_reclaim_on_the_gpu(tmp_path):
    _build()
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    for i in range(3):
        b.add_node(B.Node(f"n{i}", {"cpu": 4, "memory": 8 * G, "pods": 10}, labels={HOSTNAME: f"n{i}", ZONE: f"z{i % 2}"}))
    b.add_pod_group(B.PodGroup("ns", "run", "q", 1))
    b.add_pod_group(B.PodGroup("ns", "g", "q", 1))
    b.add_pod(B.Pod("ns", "r0", "n0", "Running", {"cpu": 1, "memory": G}, group="run", labels={"app": "web"}, uid="u-r0"))
    b.add_pod(B.Pod("ns", "p0", "", "Pending", {"cpu": 1, "memory": G}, group="g", labels={"app": "web"}, uid="u-p0",
                    pod_anti_affinity=B.PodAffinity(required=[B.PodAffinityTerm(ZONE, match_labels={"app": "web"})])))
    got = run_cases(tmp_path, b, [("c", ("reclaim", "allocate"), "cycle", PluginConf.default())])
    assert got["c"]["error"] is not None and "KB_E_UNSUPPORTED_FEATURE" in got["c"]["error"], got["c"]
