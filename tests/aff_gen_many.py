"""Seeded sessions with MANY inter-pod affinity counter groups (more than the 64 that fit the masks of kb_pod_affinity): the
generators of aff_gen.py with the app label drawn from `n_apps` values instead of four, so that the terms are mostly distinct and each
costs its own counter group.  Used by the tests of groups >= 64 (task_xgroup)."""
from __future__ import annotations

import numpy as np

from kube_batch_b200 import builder as B
from aff_gen import APPS, HOST, RACK, ZONE


def _apps(n_apps: int):
    """the app label values a generator draws from: APPS, or n_apps > 0 distinct values (many distinct terms -> many counter groups)"""
    return APPS if not n_apps else [f"app{i}" for i in range(n_apps)]


def _term(rng, hard: bool, apps=APPS) -> B.PodAffinityTerm:
    na = len(apps)
    key = [HOST, ZONE, RACK][int(rng.integers(0, 3))] if hard or rng.random() < 0.9 else ""
    t = B.PodAffinityTerm(key)
    r = rng.random()
    if r < 0.5:
        t.match_labels = {"app": apps[int(rng.integers(0, na))]}
    elif r < 0.65:
        t.match_expressions = [("app", "In", [apps[int(rng.integers(0, na))], apps[int(rng.integers(0, na))]])]
    elif r < 0.75:
        t.match_expressions = [("app", "NotIn", [apps[int(rng.integers(0, na))]])]
    elif r < 0.83:
        t.match_expressions = [("tier", "Exists", [])]
    elif r < 0.9:
        t.match_expressions = [("tier", "DoesNotExist", [])]
        t.match_labels = {"app": apps[int(rng.integers(0, na))]}
    elif r < 0.95:
        pass                                    # empty selector: everything in the namespaces
    else:
        t.nil_selector = True                   # nothing
    r = rng.random()
    if r < 0.15:
        t.namespaces = ["ns1", "ns2"]
    elif r < 0.25:
        t.namespaces = ["ns2"]
    return t


def _spec(rng, p_req=0.6, p_pref=0.5, apps=APPS):
    a = B.PodAffinity()
    if rng.random() < p_req:
        a.required = [_term(rng, True, apps) for _ in range(1 if rng.random() < 0.8 else 2)]
    if rng.random() < p_pref:
        a.preferred = [(int(rng.integers(1, 100)), _term(rng, False, apps)) for _ in range(int(rng.integers(1, 3)))]
    return a


def host_spread_session(seed: int, n_nodes: int = 12, n_groups: int = 8, pipe_geometry: bool = False, ports: bool = False,
                        n_apps: int = 0) -> B.SessionBuilder:
    """Only the commonest constraint: required anti-affinity on kubernetes.io/hostname (against the pod's own or another label),
    also on pods already running; no preferred terms, no required affinity.  The engine encodes such sessions as atoms in the
    node's port words and runs them on the persistent pipeline.  pipe_geometry: R = 3 (a scalar resource), for flatten(W=2).
    n_apps > 0: the labels come from that many values (each spread label costs two counter groups)."""
    apps = _apps(n_apps)
    na = len(apps)
    rng = np.random.default_rng(seed)
    sb = B.SessionBuilder()
    nq = int(rng.integers(1, 3))
    for q in range(nq):
        sb.add_queue(B.Queue(f"q{q}", weight=int(rng.integers(1, 4)), creation=q))
    for i in range(n_nodes):
        cpu = int(rng.choice([2, 4, 8]))
        alloc = B.build_resource_list(str(cpu), f"{cpu * 2}Gi")
        if pipe_geometry:
            alloc[B.GPU] = 4.0
        else:
            alloc.pop(B.GPU, None)
        sb.add_node(B.build_node(f"n{i:03d}", alloc, labels={HOST: f"n{i:03d}", ZONE: f"z{i % 3}"}, pods=int(rng.choice([3, 110]))))

    def anti(label):
        t = B.PodAffinityTerm(HOST, match_labels={"app": label})
        if rng.random() < 0.2:
            t.namespaces = ["ns1", "ns2"]
        return B.PodAffinity(required=[t] if rng.random() < 0.85 else [t, B.PodAffinityTerm(HOST, match_expressions=[("app", "Exists", [])])])
    uid = 0
    sb.add_pod_group(B.PodGroup("ns1", "run-a", "q0", min_member=1))
    load = {}
    for i in range(int(rng.integers(0, n_nodes))):
        host = int(rng.integers(0, n_nodes))
        if load.get(host, 0) >= 1:
            continue
        load[host] = 1
        lab = apps[int(rng.integers(0, na))]
        p = B.build_pod("ns1", f"r{i}", f"n{host:03d}", "Running", {"cpu": 1.0, "memory": 1e9}, "run-a", labels={"app": lab})
        if rng.random() < 0.5:
            p.pod_anti_affinity = anti(apps[int(rng.integers(0, na))])
        p.uid = f"u{uid:05d}"; uid += 1
        sb.add_pod(p)
    for g in range(n_groups):
        ns = "ns1" if rng.random() < 0.8 else "ns2"
        ntask = int(rng.integers(1, 7))
        sb.add_pod_group(B.PodGroup(ns, f"pg{g}", f"q{int(rng.integers(0, nq))}", min_member=int(rng.integers(1, ntask + 1)), creation=g))
        lab = apps[int(rng.integers(0, na))]
        spec = anti(lab if rng.random() < 0.7 else apps[int(rng.integers(0, na))]) if rng.random() < 0.6 else None
        req = {"cpu": float(rng.choice([0.5, 1, 2])), "memory": float(rng.choice([1, 2])) * 1e9}
        if pipe_geometry and rng.random() < 0.3:
            req[B.GPU] = 1.0
        hp = [("", "TCP", 8000 + int(rng.integers(0, 3)))] if ports and rng.random() < 0.3 else []
        for i in range(ntask):
            p = B.build_pod(ns, f"pg{g}-{i}", "", "Pending", dict(req), f"pg{g}", labels={"app": lab})
            p.pod_anti_affinity = spec
            p.host_ports = list(hp)
            p.creation = int(rng.integers(0, 3))
            p.uid = f"u{uid:05d}"; uid += 1
            sb.add_pod(p)
    return sb


def random_affinity_session(seed: int, n_nodes: int = 12, n_groups: int = 6, p_affine: float = 0.6, besteffort: bool = False,
                            n_apps: int = 0) -> B.SessionBuilder:
    """aff_gen.random_affinity_session with the app drawn from n_apps values: with ~100 PodGroups and n_apps ~ 50 the session has
    about a hundred counter groups."""
    apps = _apps(n_apps)
    na = len(apps)
    rng = np.random.default_rng(seed)
    sb = B.SessionBuilder()
    nq = int(rng.integers(1, 3))
    for q in range(nq):
        sb.add_queue(B.Queue(f"q{q}", weight=int(rng.integers(1, 4)), creation=q))
    zones = int(rng.integers(2, 4))
    for i in range(n_nodes):
        labels = {HOST: f"n{i:03d}"}
        if rng.random() < 0.9:
            labels[ZONE] = f"z{i % zones}"
        if rng.random() < 0.7:
            labels[RACK] = f"r{i % 4}"
        cpu = int(rng.choice([4, 8, 16]))
        sb.add_node(B.build_node(f"n{i:03d}", B.build_resource_list(str(cpu), f"{cpu * 2}Gi"), labels=labels, pods=int(rng.choice([4, 110]))))
    uid = 0
    # pods already running: some belong to session jobs (util.PodLister sees them), some to a group without queue (NodeInfo.Tasks only)
    sb.add_pod_group(B.PodGroup("ns1", "run-a", "q0", min_member=1))
    sb.add_pod_group(B.PodGroup("ns2", "run-b", "nosuchqueue", min_member=1))
    load = {}
    for i in range(int(rng.integers(0, n_nodes))):
        ns, grp = ("ns1", "run-a") if rng.random() < 0.7 else ("ns2", "run-b")
        host = int(rng.integers(0, n_nodes))
        if load.get(host, 0) >= 2:
            continue                      # never over-commit a node: the cache would refuse the pod (node_info.go:161-167)
        load[host] = load.get(host, 0) + 1
        p = B.build_pod(ns, f"r{i}", f"n{host:03d}", "Running", B.build_resource_list("1", "1Gi"), grp,
                        labels={"app": apps[int(rng.integers(0, na))]})
        if rng.random() < 0.3:
            p.labels["tier"] = "x"
        if rng.random() < 0.5:
            if rng.random() < 0.5:
                p.pod_affinity = _spec(rng, 0.5, 0.6, apps)
            if rng.random() < 0.6:
                p.pod_anti_affinity = _spec(rng, 0.5, 0.6, apps)
        p.uid = f"u{uid:05d}"; uid += 1
        sb.add_pod(p)
    for g in range(n_groups):
        ns = "ns1" if rng.random() < 0.7 else "ns2"
        ntask = int(rng.integers(1, 6))
        sb.add_pod_group(B.PodGroup(ns, f"pg{g}", f"q{int(rng.integers(0, nq))}", min_member=int(rng.integers(1, ntask + 1)), creation=g))
        labels = {"app": apps[int(rng.integers(0, na))]}
        if rng.random() < 0.3:
            labels["tier"] = "x"
        aff = _spec(rng, apps=apps) if rng.random() < p_affine * 0.6 else None
        anti = _spec(rng, apps=apps) if rng.random() < p_affine else None
        req = {} if (besteffort and rng.random() < 0.5) else B.build_resource_list(str(int(rng.choice([1, 2, 3]))), f"{int(rng.choice([1, 2, 4]))}Gi")
        for i in range(ntask):
            p = B.build_pod(ns, f"pg{g}-{i}", "", "Pending", req, f"pg{g}", labels=dict(labels))
            p.pod_affinity, p.pod_anti_affinity = aff, anti
            p.creation = int(rng.integers(0, 4))
            p.uid = f"u{uid:05d}"; uid += 1
            if besteffort and not req and rng.random() < 0.3:
                p.requests = {}
            sb.add_pod(p)
    return sb


def evict_spread_cluster(seed: int, members_running: bool = False, n_apps: int = 0, n_pod_groups: int = 0, W: int = 0):
    """Clusters that make reclaim / preempt evict (several queues, priorities, Running / terminating / Pending pods like
    tests/test_evict_parity.random_cluster) whose PENDING pods partly carry "one replica per host"; members_running: the pods already
    running carry the labels + terms too (then a victim can be a member of a counter group and the engine refuses the evicting actions).
    n_apps / n_pod_groups > 0: that many label values / PodGroups (instead of 3 / 2..8), for sessions with many counter groups;
    W > 0: words per port mask (room for more groups as atoms)."""
    apps = APPS[:3] if not n_apps else _apps(n_apps)
    rng = np.random.default_rng(7000 + seed)
    b = B.SessionBuilder()
    nq = int(rng.integers(1, 4))
    for q in range(nq):
        b.add_queue(B.Queue(f"q{q}", int(rng.integers(1, 4)), creation=int(rng.integers(0, 3))))
    nn = int(rng.integers(2, 9))
    for n in range(nn):
        b.add_node(B.Node(f"n{n:04d}", {"cpu": 8, "memory": 32e9, "pods": int(rng.integers(6, 14))}, labels={HOST: f"n{n:04d}"}))
    cap = {f"n{n:04d}": 8.0 for n in range(nn)}
    k = 0
    n_pg = int(rng.integers(2, 9))
    for g in range(n_pod_groups or n_pg):
        b.add_pod_group(B.PodGroup("ns", f"g{g}", f"q{int(rng.integers(0, nq))}", min_member=int(rng.integers(0, 4)),
                                   priority=int(rng.integers(0, 3)), creation=int(rng.integers(0, 4))))
        cpu = float(rng.choice([0.5, 1, 2, 3]))
        req = {"cpu": cpu, "memory": cpu * 1e9}
        lab = apps[int(rng.integers(0, len(apps)))]
        spread = rng.random() < 0.6
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
            p = B.Pod("ns", f"g{g}-p{i}", node, "Pending" if state == "Pending" else "Running", dict(req), group=f"g{g}",
                      priority=int(rng.integers(0, 3)), creation=int(rng.integers(0, 5)) if rng.random() < 0.5 else k, deleting=(state == "Deleting"))
            if spread and (state == "Pending" or members_running):
                p.labels = {"app": lab}
                p.pod_anti_affinity = B.PodAffinity(required=[B.PodAffinityTerm(HOST, match_labels={"app": lab})])
            b.add_pod(p)
            k += 1
    return b.flatten(W=W) if W else b.flatten()
