"""reclaim / preempt in sessions whose pending pods carry preferred node affinity (nodeAffinity.preferredDuringScheduling...).

preempt orders its nodes with util.PrioritizeNodes (preempt.go:180-189), and NodeAffinityPriority's NormalizeReduce divides by the max
count over util.PredicateNodes: every node that passes ssn.PredicateFn, whether or not it has Running tasks, eligible victims or
free resources, taken afresh for every preemptor.  reclaim walks ssn.Nodes in order and never scores (reclaim.go:113-115).
kb_evict.h runs a pass over all nodes for that max before the sweep of such a class; these tests check it on the CPU emulation
against the oracle (hand vectors, random clusters, host-level anti-affinity, a synthetic cluster)."""
from __future__ import annotations

import numpy as np
import pytest

from kube_batch_b200 import abi, builder as B, synth
from kube_batch_b200.snapshot import PluginConf, PluginOption
from oracle import kbo
import aff_gen
import util
from test_emu_parity import PREF_CONFS
from test_evict_parity import ACTION_LISTS, FULL_LIST, compare, tier_variants

T = True
ZONES = ("a", "b", "c")
PREF = [(100, [("zone", "In", ["a"])]), (20, [("zone", "In", ["b"])])]


# ------------------------------------------------------------------------------------------------ hand-computed vectors
def vector_tiers(weight=None, nodeorder=True) -> PluginConf:
    """priority + gang + conformance choose the victims; nodeorder (leastrequested 1, balancedresource 1, nodeaffinity `weight`) scores."""
    second = [PluginOption("predicates", enabled_predicate=T)]
    if nodeorder:
        second.append(PluginOption("nodeorder", enabled_node_order=T, arguments={} if weight is None else {"nodeaffinity.weight": str(weight)}))
    return PluginConf([[PluginOption("priority", enabled_job_order=T, enabled_task_order=T, enabled_preemptable=T),
                        PluginOption("gang", enabled_preemptable=T, enabled_reclaimable=T),
                        PluginOption("conformance", enabled_preemptable=T, enabled_reclaimable=T)], second])


def vector(a="empty", a_pods=110, a_tainted=False, b_busy=25, c_busy=1, preemptors=1, two_queues=False):
    """n-a (zone a, count 100), n-b (zone b, count 20), n-c (zone c, count 0); n-b and n-c carry two low-priority victims each.
    a: "empty" (no Running task), "full" (one Running pod of a higher-priority job takes all its cpu: no victim, no Idle) or
    "victim" (one small low-priority pod).  a_tainted: n-a fails the predicates (an untolerated NoSchedule taint), which takes its
    count out of the max.  b_busy / c_busy: cpu of the big victim on n-b / n-c, which sets the resource scores.
    two_queues: the victims' job sits in another queue (reclaim)."""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_queue(B.Queue("q2", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q2" if two_queues else "q", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "top", "q", min_member=1, priority=5))
    b.add_pod_group(B.PodGroup("ns", "hi", "q", min_member=preemptors, priority=2))
    b.add_node(B.Node("n-a", {"cpu": 64, "memory": 256e9, "pods": a_pods}, labels={"zone": "a"},
                      taints=[("dedicated", "x", "NoSchedule")] if a_tainted else []))
    b.add_node(B.Node("n-b", {"cpu": 64, "memory": 256e9, "pods": 110}, labels={"zone": "b"}))
    b.add_node(B.Node("n-c", {"cpu": 64, "memory": 256e9, "pods": 110}, labels={"zone": "c"}))
    if a == "full":
        b.add_pod(B.Pod("ns", "a-top", "n-a", "Running", {"cpu": 64, "memory": 1e9}, group="top"))
    elif a == "victim":
        b.add_pod(B.Pod("ns", "a-low", "n-a", "Running", {"cpu": 1, "memory": 1e9}, group="low"))
    b.add_pod(B.Pod("ns", "b-low", "n-b", "Running", {"cpu": b_busy, "memory": 1e9}, group="low"))
    b.add_pod(B.Pod("ns", "b-low2", "n-b", "Running", {"cpu": 1, "memory": 1e9}, group="low"))
    b.add_pod(B.Pod("ns", "c-low", "n-c", "Running", {"cpu": c_busy, "memory": 1e9}, group="low"))
    b.add_pod(B.Pod("ns", "c-low2", "n-c", "Running", {"cpu": 1, "memory": 1e9}, group="low"))
    for k in range(preemptors):
        b.add_pod(B.Pod("ns", f"p{k}", "", "Pending", {"cpu": 1, "memory": 1e9}, group="hi", creation=k, preferred_terms=PREF))
    return b.flatten()


# (name, kwargs of `vector`, tiers, action, expected nodes of the preemptors, the same with n-a tainted (None: not asked))
# Scores (leastrequested + balancedresource) with the default vector: n-b 12, n-c 18, n-a 18 (empty) / 0 (full).
VECTORS = [
    # (a) n-a has no Running task, so no key, yet it passes the predicates and holds the max count 100: n-b's term is
    #     10 * 20 / 100 = 2 and n-c (18 > 12 + 2) wins.  Out of the max (tainted), n-b's term is 10 and n-b wins (22 > 18).
    ("a: a node without victims holds the max", dict(a="empty"), vector_tiers(), "preempt", ["n-c"], ["n-b"]),
    # (b) the same with n-a full of a higher-priority pod: no Idle, no victim, still in util.PredicateNodes
    ("b: a full node still counts", dict(a="full"), vector_tiers(), "preempt", ["n-c"], ["n-b"]),
    # (c) n-a has a victim and a cap of 2 pods: p0 goes there (18 + 10), its Pipeline fills the cap, max_pods drops n-a for p1,
    #     the max falls to 20 and p1 picks n-b (12 + 10 > 18).  A max kept from p0's sweep (100) would send p1 to n-c.
    ("c: the max drops once the max node fills", dict(a="victim", a_pods=2, preemptors=2), vector_tiers(), "preempt", ["n-a", "n-b"], None),
    # (d) nodeaffinity.weight -3 with n-b nearly empty and n-c busy (resource scores 18 and 6): with n-a in the max n-b loses
    #     3 * 2 = 6 points and wins (12 > 6), without it n-b loses 3 * 10 = 30 and n-c wins
    ("d: negative nodeaffinity.weight", dict(a="empty", b_busy=1, c_busy=50), vector_tiers(-3), "preempt", ["n-b"], ["n-c"]),
    # (e) no nodeorder: every score is equal, the first valid node in name order wins whatever the terms say
    ("e: no nodeorder", dict(a="empty"), vector_tiers(nodeorder=False), "preempt", ["n-b"], ["n-b"]),
    # (f) reclaim walks ssn.Nodes in order and never scores
    ("f: reclaim ignores the terms", dict(a="empty", two_queues=True), vector_tiers(), "reclaim", ["n-b"], ["n-b"]),
]


def _picks(s, o):
    return [s.meta["nodes"][n] if n >= 0 else None for n in o.decisions["node"]]


@pytest.mark.parametrize("case", VECTORS, ids=lambda c: c[0].split(":")[0])
def test_hand_vectors_on_the_oracle(case):
    name, kw, tiers, action, want, want_tainted = case
    s = vector(**kw)
    o, ev, _ = kbo.cycle(s, tiers, actions=(action,), running=s.meta["running"])
    assert _picks(s, o) == want, name
    assert int(ev.sum()) >= 1
    if want_tainted is not None:
        st = vector(a_tainted=True, **kw)
        ot, _, _ = kbo.cycle(st, tiers, actions=(action,), running=st.meta["running"])
        assert _picks(st, ot) == want_tainted, name


@pytest.mark.parametrize("case", VECTORS, ids=lambda c: c[0].split(":")[0])
def test_hand_vectors_on_the_emulation(case):
    name, kw, tiers, action, want, want_tainted = case
    for tainted in ((False, True) if want_tainted is not None else (False,)):
        s = vector(a_tainted=tainted, **kw)
        o, ev, order = kbo.cycle(s, tiers, actions=(action,), running=s.meta["running"])
        g, gev, gorder = util.emu_evict(s, tiers, action, s.meta["running"])
        compare(f"{name} tainted={tainted}", o, ev, order, g, gev, gorder, util.emu_states(g))
        assert _picks(s, g) == (want_tainted if tainted else want), name
        g, gev, gorder = util.emu_cycle(s, tiers, (action,), s.meta["running"], mode=1)
        compare(f"{name} tainted={tainted} kb_cycle", o, ev, order, g, gev, gorder, util.emu_states(g))


# ------------------------------------------------------------------------------------------------ random clusters
def pref_cluster(seed: int, big: bool = False, spread: bool = False):
    """test_evict_parity.random_cluster with zone labels on the nodes and preferred zone terms (weights 0 / 1 / 20 / 50 / 100) on most
    pending pods.  Odd seeds use the persistent pipeline's record geometry (R = 3, W = 2), even seeds another one (R = 2, W = 1).
    spread: the pending pods of some groups also carry "one replica per host" (host-level anti-affinity, kept as atoms)."""
    rng = np.random.default_rng(9100 + seed)
    pipe = seed % 2 == 1
    b = B.SessionBuilder()
    nq = int(rng.integers(1, 4))
    for q in range(nq):
        b.add_queue(B.Queue(f"q{q}", int(rng.integers(1, 4)), creation=int(rng.integers(0, 3))))
    nn = int(rng.integers(2, 9)) if not big else int(rng.integers(150, 400))
    for n in range(nn):
        alloc = {"cpu": 8, "memory": 32e9, "pods": int(rng.integers(4, 14))}
        if pipe:
            alloc["nvidia.com/gpu"] = 4
        labels = {"zone": ZONES[int(rng.integers(0, 3))]}
        if spread:
            labels[aff_gen.HOST] = f"n{n:04d}"
        b.add_node(B.Node(f"n{n:04d}", alloc, labels=labels))
    cap = {f"n{n:04d}": 8.0 for n in range(nn)}
    k = 0
    for g in range(int(rng.integers(2, 9)) if not big else int(rng.integers(40, 90))):
        ns = "kube-system" if rng.random() < 0.1 else "ns"
        b.add_pod_group(B.PodGroup(ns, f"g{g}", f"q{int(rng.integers(0, nq))}", min_member=int(rng.integers(0, 4)),
                                   priority=int(rng.integers(0, 3)), creation=int(rng.integers(0, 4))))
        cpu = float(rng.choice([0.5, 1, 2, 3]))
        req = {"cpu": cpu, "memory": cpu * 1e9}
        pref = [(int(rng.choice([0, 1, 20, 50, 100])), [("zone", "In", [ZONES[int(rng.integers(0, 3))]])]) for _ in range(int(rng.integers(1, 4)))]
        with_pref = rng.random() < 0.8
        lab = aff_gen.APPS[int(rng.integers(0, 3))]
        with_spread = spread and rng.random() < 0.6
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
            pending = state == "Pending"
            p = B.Pod(ns, f"g{g}-p{i}", node, "Pending" if pending else "Running", dict(req), group=f"g{g}",
                      priority=int(rng.integers(0, 3)), creation=int(rng.integers(0, 5)) if rng.random() < 0.5 else k,
                      deleting=(state == "Deleting"), preferred_terms=pref if (pending and with_pref) else [])
            if with_spread and pending:
                p.labels = {"app": lab}
                p.pod_anti_affinity = B.PodAffinity(required=[B.PodAffinityTerm(aff_gen.HOST, match_labels={"app": lab})])
            b.add_pod(p)
            k += 1
    return b.flatten(W=2 if pipe else 1)


def pref_tiers():
    """tier_variants() + the PREF_CONFS weights (nodeaffinity.weight 5 / -3, no nodeorder)"""
    yield from tier_variants()
    for i, conf in enumerate(PREF_CONFS[1:]):
        yield f"pref_conf{i + 1}", conf


def strip_pref(s):
    """the same snapshot without the preferred terms"""
    import copy
    t = copy.deepcopy(s)
    t.task_flags &= ~np.uint32(abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY)
    t.task_n_pref_terms[:] = 0
    t.invalidate()
    return t


def check_cluster(s, what, lists, modes):
    for tname, tiers in pref_tiers():
        for acts in lists:
            o, ev, order = kbo.cycle(s, tiers, actions=acts, running=s.meta["running"])
            if len(acts) == 1:
                g, gev, gorder = util.emu_evict(s, tiers, acts[0], s.meta["running"])
                compare(f"{what} {tname} {acts} kb_evict", o, ev, order, g, gev, gorder, util.emu_states(g))
            for mode in modes:
                g, gev, gorder = util.emu_cycle(s, tiers, acts, s.meta["running"], mode=mode)
                w = f"{what} {tname} {acts} mode {mode}"
                compare(w, o, ev, order, g, gev, gorder, util.emu_states(g))
                util.assert_same_decisions(o.decisions, g.decisions, w)


@pytest.mark.parametrize("seed", range(24))
def test_random_clusters_on_the_emulation(seed):
    s = pref_cluster(seed)
    if not (s.task_n_pref_terms > 0).any():
        pytest.skip("no pending pod with preferred terms drawn")
    check_cluster(s, f"seed {seed}", (("reclaim",), ("preempt",)) + (ACTION_LISTS if seed % 3 == 0 else (FULL_LIST,)), (1, 5))


@pytest.mark.parametrize("seed", range(2))
def test_larger_clusters_on_the_emulation(seed):
    s = pref_cluster(100 + seed, big=True)
    check_cluster(s, f"big seed {seed}", (("preempt",), FULL_LIST), (1, 5))


def test_the_preferred_terms_move_preemptors():
    """The clusters above can fail: over them, preemptors with preferred terms land on other nodes than they would without
    the terms (i.e. than a preempt that ordered the nodes by the resource scores alone, or by name)."""
    moved = 0
    for seed in range(24):
        s = pref_cluster(seed)
        plain = strip_pref(s)
        for _, tiers in pref_tiers():
            o, _, _ = kbo.cycle(s, tiers, actions=("preempt",), running=s.meta["running"])
            p, _, _ = kbo.cycle(plain, tiers, actions=("preempt",), running=plain.meta["running"])
            pip = (o.decisions["kind"] == 2) & (s.task_n_pref_terms > 0)
            moved += int((pip & (o.decisions["node"] != p.decisions["node"])).sum())
    assert moved >= 5, moved


@pytest.mark.parametrize("seed", range(12))
def test_host_level_anti_affinity_with_preferred_terms_on_the_emulation(seed):
    """Preferred node affinity together with host-level inter-pod anti-affinity kept as atoms of the node records: the evicting
    actions run (no pod already running is a member of a counter group)."""
    s = pref_cluster(200 + seed, spread=True)
    if s.pod_affinity is None:
        pytest.skip("no spread group drawn")
    check_cluster(s, f"spread seed {seed}", (("preempt",), ("reclaim", "allocate", "backfill", "preempt"), ("allocate", "preempt")), (1,))


@pytest.mark.parametrize("seed", range(2))
def test_synthetic_cluster_with_preferred_terms_on_the_emulation(seed):
    """BASELINE-shaped synthetic session, 30 % of its PodGroups with preferred zone terms, 40 % of the filler PodGroups preemptable:
    the shipped action list evicts hundreds of pods, all of it must match."""
    s = synth.add_node_pref(synth.random_session(seed, tasks=3000, jobs=300, nodes=600, queues=3, oversub=2.0), 0.3)
    run = synth.running_of(s, 0.4)
    o, ev, order = kbo.cycle(s, PluginConf.default(), actions=FULL_LIST, running=run)
    assert int(ev.sum()) > 500
    for mode in (1, 5):
        g, gev, gorder = util.emu_cycle(s, PluginConf.default(), FULL_LIST, run, mode=mode)
        compare(f"synthetic {seed} mode {mode}", o, ev, order, g, gev, gorder, util.emu_states(g))
        util.assert_same_decisions(o.decisions, g.decisions, f"synthetic {seed} mode {mode}")


def test_add_node_pref_matches_the_flattener():
    """synth.add_node_pref fills the arrays as builder.flatten does for the same pods, and leaves synth.make alone."""
    s = synth.add_node_pref(synth.random_session(3, tasks=200, jobs=20, nodes=40), 0.5)
    has = (s.task_flags & abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY) != 0
    assert has.any() and (~has).any()
    assert ((s.task_n_pref_terms > 0) == has).all() and (s.task_n_pref_terms <= 3).all()
    for t in np.nonzero(has)[0]:
        n = int(s.task_n_pref_terms[t])
        assert set(s.task_pref_weights[:n, t].tolist()) <= {1, 10, 50, 100} and (s.task_pref_weights[n:, t] == 0).all()
        for p in range(n):
            assert int(s.task_pref_terms[p, 0, t]) in (1, 2, 4) and (s.task_pref_terms[p, 1:, t] == 0).all()
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_pod_group(B.PodGroup("ns", "g", "q"))
    b.add_node(B.Node("n0", {"cpu": 8, "memory": 8e9}, labels={"zone": "a"}))
    b.add_pod(B.Pod("ns", "p", "", "Pending", {"cpu": 1, "memory": 1e9}, group="g", preferred_terms=[(10, [("zone", "In", ["a"])])]))
    f = b.flatten()
    assert int(f.task_flags[0]) & abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY and int(f.task_n_pref_terms[0]) == 1
    assert int(f.task_pref_weights[0, 0]) == 10 and bin(int(f.task_pref_terms[0, 0, 0])).count("1") == 1
    a, _ = synth.make("c2")
    c, _ = synth.make("c2")
    synth.add_node_pref(c, 0.3)
    assert not (a.task_n_pref_terms != 0).any() and (c.task_n_pref_terms != 0).any()
