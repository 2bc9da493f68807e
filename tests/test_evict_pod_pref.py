"""reclaim / preempt in sessions whose pods carry PREFERRED inter-pod (anti)affinity (the soft spread of many Helm charts).

Such a session runs on the counter path (DESIGN 5e).  preempt orders its nodes with util.PrioritizeNodes (preempt.go:180-189), so
InterPodAffinityPriority enters the score: the weights of the pods in NodeInfo.Tasks of every node that passes ssn.PredicateFn,
normalised by the min / max count over the same nodes.  An evicted pod stays in NodeInfo.Tasks as Releasing; a Pipelined preemptor
is added (its Spec.NodeName stays "": cachedNodeInfo.GetNodeInfo's first node holding such a pod); a discarded Statement takes its
Pipelined pods out again.  The evicting actions run when no class reads a counter group in predicate step 10; every other counter-path
session is still refused.  Checked on the CPU emulation against the object-level oracle."""
from __future__ import annotations

import copy

import numpy as np
import pytest

from kube_batch_b200 import abi, builder as B, synth
from kube_batch_b200.snapshot import PluginConf, PluginOption
from oracle import kbo
import aff_gen
import util
from test_evict_parity import compare, tier_variants

T = True
HOST = aff_gen.HOST
REFUSED = "reclaim / preempt in this session with inter-pod affinity are outside this build"
LISTS = (("reclaim", "allocate", "backfill", "preempt"), ("preempt",), ("allocate", "preempt"))


# ------------------------------------------------------------------------------------------------ hand-computed vectors
def vtiers(podaff=None, nodeaff=None) -> PluginConf:
    """priority + gang + conformance choose the victims; predicates; nodeorder (leastrequested 1, balancedresource 1,
    podaffinity / nodeaffinity weights as given) scores."""
    args = {}
    if podaff is not None:
        args["podaffinity.weight"] = str(podaff)
    if nodeaff is not None:
        args["nodeaffinity.weight"] = str(nodeaff)
    return PluginConf([[PluginOption("priority", enabled_job_order=T, enabled_task_order=T, enabled_preemptable=T),
                        PluginOption("gang", enabled_preemptable=T, enabled_reclaimable=T, enabled_job_pipelined=T),
                        PluginOption("conformance", enabled_preemptable=T, enabled_reclaimable=T)],
                       [PluginOption("predicates", enabled_predicate=T), PluginOption("nodeorder", enabled_node_order=T, arguments=args)]])


def anti(w, app="web", key=HOST):
    return B.PodAffinity(preferred=[(w, B.PodAffinityTerm(key, match_labels={"app": app}))])


def vector(nodes=("n-a", "n-b", "n-c"), siblings=None, victims=None, extra=None, preemptors=1, pre_w=10, sib_w=0,
           tainted=(), full=(), low_pods=None, two_queues=False, min_member=None, pre_pref=None, zones=None, pre_anti=None):
    """Nodes of 64 cpu, one hostname each.  Every node carries a 16-cpu "top" pod (priority 5, never a victim) — labelled app=web on
    the nodes in `siblings` (a Running sibling of the preemptors, with its own soft anti-affinity of weight `sib_w` if > 0) — and a
    24-cpu low-priority victim (job "low") unless `victims` names the nodes that get one.  `extra`: (node, cpu, memory) more top pods (resource
    scores).  The preemptors (job "hi", priority 2, 1 cpu) carry app=web and soft anti-affinity of weight `pre_w` on the hostname.
    `full`: nodes whose top pod takes all 64 cpu (no victim then).  `tainted`: nodes that fail the predicates."""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_queue(B.Queue("q2", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q2" if two_queues else "q", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "top", "q", min_member=1, priority=5))
    b.add_pod_group(B.PodGroup("ns", "hi", "q", min_member=min_member or preemptors, priority=2))
    siblings = siblings or {}
    victims = nodes if victims is None else victims
    for i, n in enumerate(nodes):
        labels = {HOST: n, "zone": (zones or {}).get(n, "z")}
        b.add_node(B.Node(n, {"cpu": 64, "memory": 256e9, "pods": 110}, labels=labels,
                          taints=[("dedicated", "x", "NoSchedule")] if n in tainted else []))
        for k in range(siblings.get(n, 0) if isinstance(siblings, dict) else (1 if n in siblings else 0)):
            p = B.Pod("ns", f"{n}-web{k}", n, "Running", {"cpu": 16 if k == 0 else 0.5, "memory": 1e9}, group="top")
            p.labels = {"app": "web"}
            if sib_w:
                p.pod_anti_affinity = anti(sib_w)
            b.add_pod(p)
        has_sib = (siblings.get(n, 0) if isinstance(siblings, dict) else (n in siblings))
        if not has_sib:
            b.add_pod(B.Pod("ns", f"{n}-top", n, "Running", {"cpu": 64 if n in full else 16, "memory": 1e9}, group="top"))
        if n in victims and n not in full:
            for k in range((low_pods or {}).get(n, 1)):
                b.add_pod(B.Pod("ns", f"{n}-low{k}", n, "Running", {"cpu": 24 if k == 0 else 0.5, "memory": 1e9}, group="low"))
    for (n, cpu, mem) in (extra or ()):
        b.add_pod(B.Pod("ns", f"{n}-x{cpu}", n, "Running", {"cpu": cpu, "memory": mem}, group="top"))
    for k in range(preemptors):
        p = B.Pod("ns", f"p{k}", "", "Pending", {"cpu": 1, "memory": 1e9}, group="hi", creation=k, preferred_terms=pre_pref or [])
        p.labels = {"app": "web"}
        p.pod_anti_affinity = pre_anti if pre_anti is not None else anti(pre_w)
        b.add_pod(p)
    return b.flatten()


def picks(s, o):
    return [s.meta["nodes"][n] if n >= 0 else None for n in o.decisions["node"]]


def run_both(s, tiers, acts, what):
    """oracle and emulation (kb_evict for one action, kb_cycle in launch modes 1 and 5): identical; returns the oracle's outcome"""
    o, ev, order = kbo.cycle(s, tiers, actions=acts, running=s.meta["running"])
    if len(acts) == 1 and acts[0] in ("reclaim", "preempt"):
        g, gev, gorder = util.emu_evict(s, tiers, acts[0], s.meta["running"])
        compare(f"{what} kb_evict", o, ev, order, g, gev, gorder, util.emu_states(g))
    for mode in (1, 5):
        g, gev, gorder = util.emu_cycle(s, tiers, acts, s.meta["running"], mode=mode)
        compare(f"{what} mode {mode}", o, ev, order, g, gev, gorder, util.emu_states(g))
        util.assert_same_decisions(o.decisions, g.decisions, f"{what} mode {mode}")
    return o, ev, order


# Every node holds 16 cpu of "top" + 24 cpu of victims, so the resource scores tie unless `extra` loads a node; a tie goes to the
# lowest node name.  The preemptor p0 (app=web, soft anti-affinity w=10 on the hostname) needs 1 cpu: one victim covers it.
def test_1_soft_anti_affinity_sends_the_preemptor_away_from_its_sibling():
    # n-a holds a Running web sibling: counts n-a -10, n-b 0, n-c 0 -> min -10 / max 0 -> scores 0 / 10 / 10; n-b wins the tie with n-c.
    # With podaffinity.weight 0 the tie of the resource scores goes to n-a.
    s = vector(siblings=("n-a",))
    o, ev, _ = run_both(s, vtiers(), ("preempt",), "v1")
    assert picks(s, o) == ["n-b"] and int(ev.sum()) == 1
    o0, _, _ = run_both(s, vtiers(podaff=0), ("preempt",), "v1 weight 0")
    assert picks(s, o0) == ["n-a"]


def test_2_the_normalisation_counts_a_full_node_and_a_node_without_victims():
    # n-a: one web sibling (-10), n-b: none (0), n-d: no victim, three siblings (-30) — in util.PredicateNodes all the same.
    # n-b carries 20 more cpu: resource scores n-a 9 (leastrequested (3 + 9) / 2 = 6, balanced 3), n-b 4 ((0 + 9) / 2 = 4, 0).
    # With n-d in the min: n-a 9 + int(10 * 20 / 30) = 15, n-b 4 + 10 = 14 -> n-a.  n-d tainted (out of the set): n-a 9 + 0,
    # n-b 14 -> n-b.
    kw = dict(nodes=("n-a", "n-b", "n-d"), siblings={"n-a": 1, "n-d": 3}, victims=("n-a", "n-b"), extra=[("n-b", 20, 1e9)])
    s = vector(**kw)
    o, _, _ = run_both(s, vtiers(), ("preempt",), "v2")
    st = vector(tainted=("n-d",), **kw)
    ot, _, _ = run_both(st, vtiers(), ("preempt",), "v2 tainted")
    assert picks(s, o) == ["n-a"] and picks(st, ot) == ["n-b"]
    # a FULL node (no Idle, no victim) holds the three siblings instead: still counted
    kw2 = dict(kw, full=("n-d",))
    s2 = vector(**kw2)
    o2, _, _ = run_both(s2, vtiers(), ("preempt",), "v2 full")
    assert picks(s2, o2) == ["n-a"]


def test_3_the_first_pipeline_changes_the_second_preemptors_counts():
    # p0 goes to n-b (test 1).  Its Pipeline puts a web pod with Spec.NodeName "" into n-b's NodeInfo.Tasks; first_unbound = n-b, so
    # p1 sees -10 on n-a and -10 on n-b -> n-c.  Without the count of p0, p1 would pick n-b again.
    s = vector(siblings=("n-a",), preemptors=2)
    o, ev, _ = run_both(s, vtiers(), ("preempt",), "v3")
    assert picks(s, o) == ["n-b", "n-c"] and int(ev.sum()) == 2


def test_4_a_discarded_statement_restores_the_counts_and_first_unbound():
    # "allocate, preempt".  allocate places the web pod `alc` into n-d's Idle: first_unbound = n-d.  preempt: job "hi" needs 3
    # pods of 30 cpu (minMember 3), only n-b and n-c carry a victim.  p0: n-a -10 (sibling), n-d -20 (alc: its term and p0's),
    # n-b 0, n-c 0 -> n-b; its Pipeline moves first_unbound to n-b, where alc now counts too.  p1: n-b -40 -> n-c.  p2 finds no
    # node: the Statement is discarded, both Pipelines are undone and first_unbound goes back to n-d.  Job "hj" (q0, 30 cpu) next:
    # n-a -10, n-d -20, n-b 0, n-c 0 -> n-b.  Left at n-b, first_unbound would count alc there and send q0 to n-c.
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "top", "q", min_member=1, priority=5))
    b.add_pod_group(B.PodGroup("ns", "hi", "q", min_member=3, priority=3))
    b.add_pod_group(B.PodGroup("ns", "hj", "q", min_member=1, priority=2))
    b.add_pod_group(B.PodGroup("ns", "alc", "q", min_member=1, priority=4))
    for n in ("n-a", "n-b", "n-c", "n-d"):
        b.add_node(B.Node(n, {"cpu": 64, "memory": 256e9, "pods": 110}, labels={HOST: n}))
        t = B.Pod("ns", f"{n}-top", n, "Running", {"cpu": 16, "memory": 1e9}, group="top")
        if n == "n-a":
            t.labels = {"app": "web"}
        b.add_pod(t)
        if n in ("n-b", "n-c"):
            b.add_pod(B.Pod("ns", f"{n}-low", n, "Running", {"cpu": 30, "memory": 1e9}, group="low"))
        fill = {"n-a": 47, "n-b": 17, "n-c": 17, "n-d": 28}[n]
        b.add_pod(B.Pod("ns", f"{n}-fill", n, "Running", {"cpu": fill, "memory": 1e9}, group="top"))
    pods = [("alc", "a0", 1)] + [("hi", f"p{k}", 30) for k in range(3)] + [("hj", "q0", 30)]
    for k, (job, name, cpu) in enumerate(pods):
        p = B.Pod("ns", name, "", "Pending", {"cpu": cpu, "memory": 1e9}, group=job, creation=k)
        p.labels = {"app": "web"}
        p.pod_anti_affinity = anti(10)
        b.add_pod(p)
    s = b.flatten()
    o, ev, _ = run_both(s, vtiers(), ("allocate", "preempt"), "v4")
    got = dict(zip(s.meta["tasks"], picks(s, o)))
    kinds = dict(zip(s.meta["tasks"], o.decisions["kind"].tolist()))
    assert got["ns/a0"] == "n-d" and kinds["ns/a0"] == abi.KB_KIND_ALLOCATED, got
    assert all(kinds[f"ns/p{k}"] not in (abi.KB_KIND_ALLOCATED, abi.KB_KIND_PIPELINED) for k in range(3)), kinds
    assert got["ns/q0"] == "n-b" and kinds["ns/q0"] == abi.KB_KIND_PIPELINED, got
    assert int(ev.sum()) == 1


def test_5_an_evicted_pod_with_terms_still_counts_as_releasing():
    # n-a and n-b each hold a low-priority victim labelled app=web with its own soft anti-affinity (w=40); n-a also a plain victim
    # of higher pod priority (popped after it).  p0: n-a and n-b both count -(10 + 40) = -50, the resource scores tie -> n-a; it
    # evicts the web victim (it covers 1 cpu).  p1: the evicted web pod stays in n-a's NodeInfo.Tasks as Releasing (-50) and p0
    # is Pipelined there (first_unbound n-a: -(10 + 10) = -20) -> n-a -70, n-b -50 -> scores 0 / 2 -> n-b.  A count that dropped
    # the evicted pod would give n-a -20 and send p1 to n-a's plain victim.
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "top", "q", min_member=1, priority=5))
    b.add_pod_group(B.PodGroup("ns", "hi", "q", min_member=1, priority=2))
    for n in ("n-a", "n-b"):
        b.add_node(B.Node(n, {"cpu": 64, "memory": 256e9, "pods": 110}, labels={HOST: n}))
        b.add_pod(B.Pod("ns", f"{n}-top", n, "Running", {"cpu": 16, "memory": 1e9}, group="top"))
        v = B.Pod("ns", f"{n}-low", n, "Running", {"cpu": 24, "memory": 1e9}, group="low", priority=0)
        v.labels = {"app": "web"}
        v.pod_anti_affinity = anti(40)
        b.add_pod(v)
    b.add_pod(B.Pod("ns", "n-a-plain", "n-a", "Running", {"cpu": 2, "memory": 1e9}, group="low", priority=1))
    for k in range(2):
        p = B.Pod("ns", f"p{k}", "", "Pending", {"cpu": 1, "memory": 1e9}, group="hi", creation=k)
        p.labels = {"app": "web"}
        p.pod_anti_affinity = anti(10)
        b.add_pod(p)
    s = b.flatten()
    o, ev, _ = run_both(s, vtiers(), ("preempt",), "v5")
    assert picks(s, o) == ["n-a", "n-b"]
    names = [f"{s.meta['nodes'][int(n)]}" for n in s.meta["running"]["node"]]
    assert int(ev.sum()) == 2 and not ev[[i for i, n in enumerate(names) if n == "n-a"]].all()


def test_6_allocate_sees_reclaims_pipelined_pods():
    # reclaim (ssn.Nodes in order, no score) pipelines p0 (20 cpu, queue q) onto n-a over the victim of queue q2; p1 (job hj, queue
    # q) finds no victim of another queue left and stays Pending.  allocate places p1 into Idle; the nodes are loaded alike (60 cpu
    # requested each), so the resource scores tie.  Its InterPodAffinityPriority counts p0 (Spec.NodeName "": first_unbound = n-a)
    # and the web sibling on n-c: n-a -20, n-b 0, n-c -10 -> n-b.  Without p0 counted, n-a would win the tie.
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_queue(B.Queue("q2", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q2", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "top", "q", min_member=1, priority=5))
    b.add_pod_group(B.PodGroup("ns", "hi", "q", min_member=1, priority=2))
    b.add_pod_group(B.PodGroup("ns", "hj", "q", min_member=1, priority=1))
    for n in ("n-a", "n-b", "n-c"):
        b.add_node(B.Node(n, {"cpu": 64, "memory": 256e9, "pods": 110}, labels={HOST: n}))
        t = B.Pod("ns", f"{n}-top", n, "Running", {"cpu": 16, "memory": 1e9}, group="top")
        if n == "n-c":
            t.labels = {"app": "web"}
        b.add_pod(t)
        if n == "n-a":
            b.add_pod(B.Pod("ns", "n-a-low", n, "Running", {"cpu": 24, "memory": 1e9}, group="low"))
        else:
            b.add_pod(B.Pod("ns", f"{n}-big", n, "Running", {"cpu": 44, "memory": 1e9}, group="top"))
    for k, (job, cpu) in enumerate((("hi", 20), ("hj", 1))):
        p = B.Pod("ns", f"p{k}", "", "Pending", {"cpu": cpu, "memory": 1e9}, group=job, creation=k)
        p.labels = {"app": "web"}
        p.pod_anti_affinity = anti(10)
        b.add_pod(p)
    s = b.flatten()
    o, ev, _ = run_both(s, vtiers(), ("reclaim", "allocate"), "v6")
    got = picks(s, o)
    assert o.decisions["kind"][0] == abi.KB_KIND_PIPELINED and got[0] == "n-a", got
    assert o.decisions["kind"][1] == abi.KB_KIND_ALLOCATED and got[1] == "n-b", got
    o0, _, _ = run_both(s, vtiers(podaff=0), ("reclaim", "allocate"), "v6 weight 0")
    assert picks(s, o0)[1] == "n-a"


def test_7_negative_weight_and_truncation_with_a_negative_minimum():
    # One web sibling on n-a, two on n-b: counts -10 / -20 / 0 -> min -20, max 0 -> scores int(10 * 10 / 20) = 5 / 0 / 10.
    # podaffinity.weight -3 subtracts them: -15 / 0 / -30 on tied resource scores -> n-b, the node with the most siblings.
    s = vector(siblings={"n-a": 1, "n-b": 2})
    o, _, _ = run_both(s, vtiers(podaff=-3), ("preempt",), "v7")
    assert picks(s, o) == ["n-b"]
    # Three siblings on n-b: min -30 -> n-a scores int(10 * 20 / 30) = int(6.67) = 6, n-c 10.  n-c carries 16 more cpu: resource
    # scores n-a 9, n-c 6 -> n-a 15, n-c 16 -> n-c.  A rounded score (7) would tie at 16 and give n-a.
    s3 = vector(siblings={"n-a": 1, "n-b": 3}, extra=[("n-c", 16, 1e9)])
    o3, _, _ = run_both(s3, vtiers(), ("preempt",), "v7 truncation")
    assert picks(s3, o3) == ["n-c"]


def test_8_together_with_preferred_node_affinity():
    # n-a: sibling (-10), zone a (node-affinity count 100); n-b: zone b (20); n-c: zone c (0).  Inter-pod scores 0 / 10 / 10,
    # node-affinity scores 10 / 2 / 0: n-a 10, n-b 12, n-c 10 -> n-b.  pmax is reduced in the same pass as the inter-pod min / max.
    pref = [(100, [("zone", "In", ["a"])]), (20, [("zone", "In", ["b"])])]
    s = vector(siblings=("n-a",), pre_pref=pref, zones={"n-a": "a", "n-b": "b", "n-c": "c"})
    o, _, _ = run_both(s, vtiers(), ("preempt",), "v8")
    assert picks(s, o) == ["n-b"]
    o2, _, _ = run_both(s, vtiers(podaff=0), ("preempt",), "v8 no inter-pod")
    assert picks(s, o2) == ["n-a"]


# ------------------------------------------------------------------------------------------------ random clusters
TOPO = (HOST, "zone")


def pod_pref_cluster(seed: int, members: bool = False):
    """Clusters that make reclaim / preempt evict (several queues, priorities, Running / terminating / Pending pods, like
    aff_gen.evict_spread_cluster) whose pods, pending and Running alike, partly carry preferred inter-pod terms at random topology
    keys (hostname / zone): soft anti-affinity and soft affinity towards one of three apps.  Some Running pods also own a
    required anti-affinity term {role=solo} that no pending pod matches.  members: some PodGroups also carry "one replica per host"
    as a REQUIRED term, Running pods included (counter groups with Running members; only sessions without the predicates plugin,
    which then read no group, may evict them)."""
    rng = np.random.default_rng(12000 + seed)
    b = B.SessionBuilder()
    nq = int(rng.integers(1, 4))
    for q in range(nq):
        b.add_queue(B.Queue(f"q{q}", int(rng.integers(1, 4)), creation=int(rng.integers(0, 3))))
    nn = int(rng.integers(2, 9))
    for n in range(nn):
        b.add_node(B.Node(f"n{n:04d}", {"cpu": 8, "memory": 32e9, "pods": int(rng.integers(5, 14))},
                          labels={HOST: f"n{n:04d}", "zone": "ab"[int(rng.integers(0, 2))]}))
    cap = {f"n{n:04d}": 8.0 for n in range(nn)}
    k = 0
    for g in range(int(rng.integers(2, 9))):
        b.add_pod_group(B.PodGroup("ns", f"g{g}", f"q{int(rng.integers(0, nq))}", min_member=int(rng.integers(0, 4)),
                                   priority=int(rng.integers(0, 3)), creation=int(rng.integers(0, 4))))
        cpu = float(rng.choice([0.5, 1, 2, 3]))
        req = {"cpu": cpu, "memory": cpu * 1e9}
        lab = aff_gen.APPS[int(rng.integers(0, 3))]
        soft = rng.random() < 0.7
        terms = []
        for _ in range(int(rng.integers(1, 3))):
            terms.append((int(rng.choice([1, 5, 20, 100])), B.PodAffinityTerm(TOPO[int(rng.integers(0, 2))],
                                                                               match_labels={"app": aff_gen.APPS[int(rng.integers(0, 3))]})))
        affine = rng.random() < 0.3
        spread = members and rng.random() < 0.5
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
                      priority=int(rng.integers(0, 3)), creation=int(rng.integers(0, 5)) if rng.random() < 0.5 else k,
                      deleting=(state == "Deleting"))
            if soft:
                p.labels = {"app": lab}
                if affine:
                    p.pod_affinity = B.PodAffinity(preferred=list(terms))
                else:
                    p.pod_anti_affinity = B.PodAffinity(preferred=list(terms))
            if spread:
                p.labels = {"app": lab}
                pa = p.pod_anti_affinity or B.PodAffinity()
                p.pod_anti_affinity = B.PodAffinity(required=[B.PodAffinityTerm(HOST, match_labels={"app": lab})], preferred=pa.preferred)
            elif state != "Pending" and rng.random() < 0.3:
                p.labels = dict(p.labels or {}, role="solo")
                pa = p.pod_anti_affinity or B.PodAffinity()
                p.pod_anti_affinity = B.PodAffinity(required=[B.PodAffinityTerm(HOST, match_labels={"role": "solo"})], preferred=pa.preferred)
            b.add_pod(p)
            k += 1
    return b.flatten()


def has_weights(s):
    return s.pod_affinity is not None and int(s.pod_affinity["n_weights"]) > 0


def check_cluster(s, what, confs, lists=LISTS):
    for tname, tiers in confs:
        for acts in lists:
            run_both(s, tiers, acts, f"{what} {tname} {acts}")


@pytest.mark.parametrize("seed", range(24))
def test_random_clusters_on_the_emulation(seed):
    s = pod_pref_cluster(seed)
    if not has_weights(s):
        pytest.skip("no preferred inter-pod term drawn")
    check_cluster(s, f"seed {seed}", list(tier_variants()) + [("podaff-3", vtiers(podaff=-3))])


def no_predicates_tiers():
    yield "no_predicates", PluginConf([[PluginOption("priority", enabled_job_order=T, enabled_task_order=T, enabled_preemptable=T),
                                        PluginOption("gang", enabled_job_order=T, enabled_job_ready=T, enabled_preemptable=T, enabled_reclaimable=T),
                                        PluginOption("conformance", enabled_preemptable=T, enabled_reclaimable=T)],
                                       [PluginOption("proportion", enabled_queue_order=T, enabled_reclaimable=T), PluginOption("nodeorder", enabled_node_order=T)]])


def test_members_of_unread_groups_are_evicted_without_withholding():
    """Counter groups nobody reads (no predicates plugin) with Running members: the evicting actions run, evict members (before, the
    eviction of a KB_RUNNING_AFF_MEMBER withheld the outcome), and the outcome equals the oracle's."""
    evicted_members = 0
    for seed in range(24):
        s = pod_pref_cluster(seed, members=True)
        if not has_weights(s):
            continue
        member = (s.meta["running"]["flags"] & abi.KB_RUNNING_AFF_MEMBER) != 0
        for tname, tiers in no_predicates_tiers():
            for acts in LISTS:
                _, ev, _ = run_both(s, tiers, acts, f"members seed {seed} {tname} {acts}")
                evicted_members += int((ev & member).sum())
    assert evicted_members >= 3, evicted_members


def test_the_inter_pod_priority_moves_preemptors():
    """Over the random clusters, some preemptors land on another node than with podaffinity.weight 0."""
    moved = 0
    for seed in range(48):
        s = pod_pref_cluster(seed)
        if not has_weights(s):
            continue
        for tname, tiers in tier_variants():
            zero = copy.deepcopy(tiers)
            for tier in zero.tiers:
                for opt in tier:
                    if opt.name == "nodeorder":
                        opt.arguments = dict(opt.arguments, **{"podaffinity.weight": "0"})
            o, _, _ = kbo.cycle(s, tiers, actions=("preempt",), running=s.meta["running"])
            z, _, _ = kbo.cycle(s, zero, actions=("preempt",), running=s.meta["running"])
            pip = o.decisions["kind"] == abi.KB_KIND_PIPELINED
            moved += int((pip & (o.decisions["node"] != z.decisions["node"])).sum())
    assert moved >= 5, moved


# ------------------------------------------------------------------------------------------------ refusals that stay
def test_a_class_that_reads_a_group_is_still_refused():
    sb = aff_gen.random_affinity_session(77, n_nodes=20, n_groups=10)
    s = sb.flatten()
    assert (s.pod_affinity["task_forbid"] != 0).any()
    for acts in (("preempt",), ("reclaim", "allocate", "backfill", "preempt")):
        with pytest.raises(RuntimeError, match=REFUSED):
            util.emu_cycle(s, PluginConf.default(), acts, s.meta["running"], mode=1)
    # a soft-spread cluster whose pending pods also carry a required anti-affinity term (forbid bits) with the predicates on
    s = pod_pref_cluster(3, members=True)
    if (s.pod_affinity["task_forbid"] != 0).any() and len(s.meta["running"]["node"]):
        with pytest.raises(RuntimeError, match=REFUSED):
            util.emu_cycle(s, PluginConf.default(), ("preempt",), s.meta["running"], mode=1)


# ------------------------------------------------------------------------------------------------ synth.add_pod_pref
def test_add_pod_pref_matches_the_flattener():
    """synth.add_pod_pref fills kb_pod_affinity as builder.flatten does for the same pods."""
    plain = B.SessionBuilder()
    groups = [("g0", 3), ("g1", 2), ("g2", 4), ("g3", 1), ("g4", 2), ("g5", 3)]
    nodes = [f"n{i}" for i in range(5)]

    def make(spec):
        b = B.SessionBuilder()
        b.add_queue(B.Queue("q", 1))
        for n in nodes:
            b.add_node(B.Node(n, {"cpu": 8, "memory": 8e9}, labels={HOST: n}))
        for gi, (g, n_pods) in enumerate(groups):
            b.add_pod_group(B.PodGroup("ns", g, "q"))
            for i in range(n_pods):
                p = B.Pod("ns", f"{g}-{i}", "", "Pending", {"cpu": 1, "memory": 1e9}, group=g, creation=gi * 10 + i)
                if spec and spec[gi] is not None:
                    lab, w = spec[gi]
                    p.labels = {"app": f"l{lab}"}
                    p.pod_anti_affinity = anti(w, app=f"l{lab}")
                b.add_pod(p)
        return b.flatten()

    del plain
    s = make(None)
    synth.add_pod_pref(s, 0.7, labels=2, seed=5)
    kinds = s.meta["pod_pref_kinds"]
    spec = []
    for j in range(s.J):
        k = int(s.pod_affinity["task_kind"][int(s.job_task_off[j])])
        spec.append(kinds[k] if k >= 0 else None)
    assert sum(x is not None for x in spec) >= 3 and len(kinds) >= 2
    f = make(spec)
    a, r = s.pod_affinity, f.pod_affinity
    for key in ("n_keysets", "n_groups", "n_kinds", "n_weights", "first_unbound_node"):
        assert int(a[key]) == int(r[key]), key
    for key in ("node_domain", "keyset_domains", "task_forbid", "task_need", "task_contrib", "task_kind", "node_kind_count0",
                "kind_unbound", "task_weight_off", "weight_kind", "weight_keyset", "weight_value"):
        np.testing.assert_array_equal(np.asarray(a[key]).reshape(-1), np.asarray(r[key]).reshape(-1), err_msg=key)
    assert ((s.task_flags & abi.KB_TASK_HAS_POD_AFFINITY) == (f.task_flags & abi.KB_TASK_HAS_POD_AFFINITY)).all()


def test_synthetic_cluster_with_soft_spread_on_the_emulation():
    """BASELINE-shaped synthetic session, 20 % of its PodGroups with soft hostname anti-affinity (synth.add_pod_pref), 40 % of the
    filler PodGroups preemptable: the shipped action list runs on the counter path and evicts.  The object-level oracle needs the
    pod objects, which a synthetic session does not have: the two launch modes of the emulation must agree, and preemptors of the
    soft-spread PodGroups must be placed."""
    s = synth.add_pod_pref(synth.random_session(4, tasks=1500, jobs=150, nodes=300, queues=3, oversub=2.0), 0.2)
    run = synth.running_of(s, 0.4)
    acts = ("reclaim", "allocate", "backfill", "preempt")
    g1, ev1, or1 = util.emu_cycle(s, PluginConf.default(), acts, run, mode=1)
    g5, ev5, or5 = util.emu_cycle(s, PluginConf.default(), acts, run, mode=5)
    compare("synthetic mode 5 vs mode 1", g1, ev1, or1, g5, ev5, or5, util.emu_states(g5))
    assert int(ev1.sum()) > 100
    soft = s.pod_affinity["task_kind"][:s.T] >= 0
    assert ((g1.decisions["kind"] == abi.KB_KIND_PIPELINED) & soft).sum() > 0
