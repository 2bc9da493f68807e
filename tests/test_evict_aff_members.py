"""reclaim / preempt evicting members of host-level anti-affinity groups ("one replica per host").

With kb_running.aff_group_off / aff_group the engine knows which counter groups every Running task is a member of.  kb_evict_build.h
keeps a member count per (atom, node) for the atoms some Running task belongs to, evict_apply lowers it when a member is evicted
(util.PodLister stops listing a Releasing pod, plugins/util/util.go:37-59) and raises it again when a discarded Statement brings
the member back; the atom's bit in the node record follows count > 0.  Tasks an earlier allocate / backfill of the cycle Allocated
are members too and are folded into the counts when an evicting action starts.

The object-level oracle lists the Running tasks of kbo_running as static pods, so an evicted member stays listed there.  The
reference drops it (util.PodLister lists AllocatedStatus tasks only): tests/follow_oracle.py builds the same oracle with the listing
following the Running tasks' status, and every result here is checked bit-exactly against it.  The hand vectors also write the
reference's placements out."""
from __future__ import annotations

import copy

import numpy as np
import pytest

from kube_batch_b200 import abi, builder as B, synth
from kube_batch_b200.snapshot import PluginConf, PluginOption
from oracle import kbo
import aff_gen
import aff_gen_many
import follow_oracle
import util
from test_evict_parity import compare, tier_variants
from test_many_aff_groups import atoms_fit

HOST = aff_gen.HOST
T = True
LISTS = (("reclaim", "allocate", "backfill", "preempt"), ("preempt",), ("allocate", "preempt"))


def with_lists(s):
    """the Running table with builder.py's group lists merged in"""
    return dict(s.meta["running"], **s.meta["running_aff_groups"])


def tiers(nodeorder=False) -> PluginConf:
    """priority + gang + conformance choose the victims; no node scores: preempt takes the first valid node in name order"""
    second = [PluginOption("predicates", enabled_predicate=T)]
    if nodeorder:
        second.append(PluginOption("nodeorder", enabled_node_order=T))
    return PluginConf([[PluginOption("priority", enabled_job_order=T, enabled_task_order=T, enabled_preemptable=T),
                        PluginOption("gang", enabled_job_pipelined=T, enabled_preemptable=T, enabled_reclaimable=T),
                        PluginOption("conformance", enabled_preemptable=T, enabled_reclaimable=T)], second])


def web_anti():
    return B.PodAffinity(required=[B.PodAffinityTerm(HOST, match_labels={"app": "web"})])


def pod(name, node, cpu, group, labels=None, anti=None, creation=0):
    p = B.Pod("ns", name, node, "Running" if node else "Pending", {"cpu": cpu, "memory": 1e9}, group=group, creation=creation)
    p.labels = dict(labels or {})
    p.pod_anti_affinity = anti
    return p


# ------------------------------------------------------------------------------------------------ hand-computed vectors
def reclaim_vector(a_pods):
    """n-a (4 cpu) carries `a_pods` (Running, queue q2, priority 0); n-b (4 cpu) is full with a pod of the reclaimers' own queue, so
    it has no victim.  r0 (no labels, 2 cpu, job hi0) and then r1 (app=web with the "one web per host" term, 2 cpu, job hi1) reclaim
    from queue q; reclaim evicts n-a's victims in UID order (names a1.. first)."""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_queue(B.Queue("q2", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q2", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "top", "q", min_member=1, priority=5))
    b.add_pod_group(B.PodGroup("ns", "hi0", "q", min_member=1, priority=3))
    b.add_pod_group(B.PodGroup("ns", "hi1", "q", min_member=1, priority=2))
    for n in ("n-a", "n-b"):
        b.add_node(B.Node(n, {"cpu": 4, "memory": 64e9, "pods": 110}, labels={HOST: n}))
    for p in a_pods:
        b.add_pod(p)
    b.add_pod(pod("b-top", "n-b", 4, "top"))
    b.add_pod(pod("r0", "", 2, "hi0"))
    b.add_pod(pod("r1", "", 2, "hi1", {"app": "web"}, web_anti()))
    return b.flatten()


def v1_only_member_evicted():
    return reclaim_vector([pod("a1-web", "n-a", 2, "low", {"app": "web"}, web_anti()), pod("a2-fill", "n-a", 2, "low")])


def v2_one_of_two_members_evicted():
    return reclaim_vector([pod("a1-web", "n-a", 2, "low", {"app": "web"}, web_anti()), pod("a2-fill", "n-a", 1, "low"),
                           pod("a3-web", "n-a", 1, "low", {"app": "web"}, web_anti())])


def v5_session():
    """a1-guard carries app=db and OWNS the term {app=web, hostname}: r1 (app=web, no term of its own) is kept off n-a by
    satisfiesExistingPodsAntiAffinity only, until the owner leaves util.PodLister"""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_queue(B.Queue("q2", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q2", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "top", "q", min_member=1, priority=5))
    b.add_pod_group(B.PodGroup("ns", "hi0", "q", min_member=1, priority=3))
    b.add_pod_group(B.PodGroup("ns", "hi1", "q", min_member=1, priority=2))
    for n in ("n-a", "n-b"):
        b.add_node(B.Node(n, {"cpu": 4, "memory": 64e9, "pods": 110}, labels={HOST: n}))
    b.add_pod(pod("a1-guard", "n-a", 2, "low", {"app": "db"}, web_anti()))
    b.add_pod(pod("a2-fill", "n-a", 2, "low"))
    b.add_pod(pod("b-top", "n-b", 4, "top"))
    b.add_pod(pod("r0", "", 2, "hi0"))
    b.add_pod(pod("r1", "", 2, "hi1", {"app": "web"}))
    return b.flatten()


def v3_discarded_statement():
    """preempt, one queue: job hi (priority 2, MinAvailable 2) has p0 (4 cpu) and p1 (100 cpu: fits nowhere).  p0 evicts a1-web, the
    only member on n-a, inside the Statement; p1 finds no node, hi is not pipelined and the Statement is discarded — a1-web is back.
    Then p2 (job hi2, priority 1, app=web with the term) must not get n-a: it takes n-b from b1-fill."""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "hi", "q", min_member=2, priority=2))
    b.add_pod_group(B.PodGroup("ns", "hi2", "q", min_member=1, priority=1))
    for n in ("n-a", "n-b"):
        b.add_node(B.Node(n, {"cpu": 4, "memory": 64e9, "pods": 110}, labels={HOST: n}))
    b.add_pod(pod("a1-web", "n-a", 4, "low", {"app": "web"}, web_anti()))
    b.add_pod(pod("b1-fill", "n-b", 4, "low"))
    b.add_pod(pod("p0", "", 4, "hi", creation=0))
    b.add_pod(pod("p1", "", 100, "hi", creation=1))
    b.add_pod(pod("p2", "", 4, "hi2", {"app": "web"}, web_anti()))
    return b.flatten()


def v4_allocate_then_preempt():
    """"allocate, preempt", one queue.  n-a (6 cpu): a1-web (app=web, no term, created last: preempt's first victim) and a2-fill, 2 cpu
    free; n-b (4 cpu) full with b1-fill.  allocate puts w0 (app=web, no term, job wj) on n-a: a member of the group of p's own term
    list.  preempt: pp (job hi) evicts a1-web on n-a — w0 is still there, so n-a stays closed for p (app=web + term, job hi2), which
    takes n-b from b1-fill.  Without w0 in the count p would get n-a (victim a2-fill)."""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "wj", "q", min_member=1, priority=3))
    b.add_pod_group(B.PodGroup("ns", "hi", "q", min_member=1, priority=2))
    b.add_pod_group(B.PodGroup("ns", "hi2", "q", min_member=1, priority=1))
    b.add_node(B.Node("n-a", {"cpu": 6, "memory": 64e9, "pods": 110}, labels={HOST: "n-a"}))
    b.add_node(B.Node("n-b", {"cpu": 4, "memory": 64e9, "pods": 110}, labels={HOST: "n-b"}))
    b.add_pod(pod("a1-web", "n-a", 2, "low", {"app": "web"}, creation=5))
    b.add_pod(pod("a2-fill", "n-a", 2, "low", creation=0))
    b.add_pod(pod("b1-fill", "n-b", 4, "low"))
    b.add_pod(pod("w0", "", 2, "wj", {"app": "web"}))
    b.add_pod(pod("pp", "", 2, "hi"))
    b.add_pod(pod("p", "", 2, "hi2", {"app": "web"}, web_anti()))
    return b.flatten()


def v6_fold_after_an_earlier_evicting_action():
    """v4 behind a reclaim that pipelines first: n-0 (2 cpu, first in name order) carries c1 (queue q); r (queue q2) reclaims it, so
    the step counter has moved before allocate places w0 on n-a.  preempt, the second evicting action of the cycle, must still count
    w0 as a member of n-a: pp evicts a1-web there and p takes n-b."""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_queue(B.Queue("q2", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "wj", "q", min_member=1, priority=3))
    b.add_pod_group(B.PodGroup("ns", "hi", "q", min_member=1, priority=2))
    b.add_pod_group(B.PodGroup("ns", "hi2", "q", min_member=1, priority=1))
    b.add_pod_group(B.PodGroup("ns", "rj", "q2", min_member=1, priority=0))
    b.add_node(B.Node("n-0", {"cpu": 2, "memory": 64e9, "pods": 110}, labels={HOST: "n-0"}))
    b.add_node(B.Node("n-a", {"cpu": 6, "memory": 64e9, "pods": 110}, labels={HOST: "n-a"}))
    b.add_node(B.Node("n-b", {"cpu": 4, "memory": 64e9, "pods": 110}, labels={HOST: "n-b"}))
    b.add_pod(pod("c1", "n-0", 2, "low"))
    b.add_pod(pod("a1-web", "n-a", 2, "low", {"app": "web"}, creation=5))
    b.add_pod(pod("a2-fill", "n-a", 2, "low", creation=0))
    b.add_pod(pod("b1-fill", "n-b", 4, "low"))
    b.add_pod(pod("w0", "", 2, "wj", {"app": "web"}))
    b.add_pod(pod("pp", "", 2, "hi"))
    b.add_pod(pod("p", "", 2, "hi2", {"app": "web"}, web_anti()))
    b.add_pod(pod("r", "", 2, "rj"))
    return b.flatten()


DECOYS = 40


def v7_atom_in_the_second_port_word():
    """v1 with 40 "one replica per host" decoy apps pending in a third queue (100 cpu: they fit nowhere): 82 counter groups, and the
    groups of a1-web come after the decoys' — their atoms sit in the second port word (W = 2)"""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_queue(B.Queue("q2", 1))
    b.add_queue(B.Queue("q3", 1))
    b.add_pod_group(B.PodGroup("ns", "low", "q2", min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "top", "q", min_member=1, priority=5))
    b.add_pod_group(B.PodGroup("ns", "hi0", "q", min_member=1, priority=3))
    b.add_pod_group(B.PodGroup("ns", "hi1", "q", min_member=1, priority=2))
    b.add_pod_group(B.PodGroup("ns", "decoy", "q3", min_member=1, priority=0))
    for n in ("n-a", "n-b"):
        b.add_node(B.Node(n, {"cpu": 4, "memory": 64e9, "pods": 110}, labels={HOST: n}))
    b.add_pod(pod("a1-web", "n-a", 2, "low", {"app": "web"}, web_anti()))
    b.add_pod(pod("a2-fill", "n-a", 2, "low"))
    b.add_pod(pod("b-top", "n-b", 4, "top"))
    for k in range(DECOYS):
        b.add_pod(pod(f"d{k:02d}", "", 100, "decoy", {"app": f"d{k}"},
                      B.PodAffinity(required=[B.PodAffinityTerm(HOST, match_labels={"app": f"d{k}"})]), creation=k))
    b.add_pod(pod("r0", "", 2, "hi0"))
    b.add_pod(pod("r1", "", 2, "hi1", {"app": "web"}, web_anti()))
    return b.flatten(W=2)


# (name, session, action list, expected node per task in task order (None: not placed), expected evicted pods in eviction order,
#  whether the oracle agrees)
VECTORS = [
    ("1: the only member on n-a is evicted, n-a opens for r1", v1_only_member_evicted, ("reclaim",),
     {"ns/r0": "n-a", "ns/r1": "n-a"}, ["ns/a1-web", "ns/a2-fill"], False),
    ("2: one of two members is evicted, n-a stays closed", v2_one_of_two_members_evicted, ("reclaim",),
     {"ns/r0": "n-a", "ns/r1": None}, ["ns/a1-web"], True),
    ("3: a discarded Statement brings the member back", v3_discarded_statement, ("preempt",),
     {"ns/p0": None, "ns/p1": None, "ns/p2": "n-b"}, ["ns/b1-fill"], True),
    ("4: a member allocate placed keeps n-a closed", v4_allocate_then_preempt, ("allocate", "preempt"),
     {"ns/w0": "n-a", "ns/pp": "n-a", "ns/p": "n-b"}, ["ns/a1-web", "ns/b1-fill"], True),
    ("5: the owner of the term is evicted, n-a opens", v5_session, ("reclaim",),
     {"ns/r0": "n-a", "ns/r1": "n-a"}, ["ns/a1-guard", "ns/a2-fill"], False),
    ("6: a member allocate placed after an earlier eviction keeps n-a closed", v6_fold_after_an_earlier_evicting_action,
     ("reclaim", "allocate", "backfill", "preempt"),
     {"ns/w0": "n-a", "ns/pp": "n-a", "ns/p": "n-b", "ns/r": "n-0"}, ["ns/c1", "ns/a1-web", "ns/b1-fill"], True),
    ("7: the only member is evicted, its atoms in the second port word", v7_atom_in_the_second_port_word, ("reclaim",),
     dict({f"ns/d{k:02d}": None for k in range(DECOYS)}, **{"ns/r0": "n-a", "ns/r1": "n-a"}), ["ns/a1-web", "ns/a2-fill"], False),
]


def placements(s, o):
    return {t: (s.meta["nodes"][n] if n >= 0 else None) for t, n in zip(s.meta["tasks"], o.decisions["node"].tolist())}


def evicted_names(s, ev, order):
    names = s.meta["running"]["names"]
    return [names[i] for i in sorted(np.nonzero(ev)[0], key=lambda i: int(order[i]))]


@pytest.mark.parametrize("case", VECTORS, ids=lambda c: c[0].split(":")[0])
def test_hand_vectors(case):
    name, make, acts, want, want_ev, oracle_agrees = case
    s = make()
    run = with_lists(s)
    assert (s.meta["running"]["flags"] & abi.KB_RUNNING_AFF_MEMBER).any() and s.pod_affinity is not None
    g, gev, gorder = util.emu_cycle(s, tiers(), acts, run, mode=1)
    assert placements(s, g) == want, name
    assert evicted_names(s, gev, gorder) == want_ev, name
    if len(acts) == 1:                                               # kbemu_evict: the action alone, from the loaded state
        e, eev, eorder = util.emu_evict(s, tiers(), acts[0], run)
        compare(name, g, gev, gorder, e, eev, eorder)
    f, fev, forder = follow_oracle.cycle(s, tiers(), acts, run)
    compare(name, f, fev, forder, g, gev, gorder, util.emu_states(g))
    o, ev, order = kbo.cycle(s, tiers(), actions=acts, running=run)
    if oracle_agrees:
        compare(name, o, ev, order, g, gev, gorder, util.emu_states(g))
    else:                                                            # the plain oracle keeps the evicted member listed: r1 finds no node
        assert placements(s, o)["ns/r1"] is None
    # without the lists the same cycle is withheld once a member is evicted
    if any(n in want_ev for n in np.array(s.meta["running"]["names"])[(s.meta["running"]["flags"] & abi.KB_RUNNING_AFF_MEMBER) != 0]):
        with pytest.raises(RuntimeError, match="withheld"):
            util.emu_cycle(s, tiers(), acts, s.meta["running"], mode=1)


def test_vector_7_puts_the_member_atoms_past_the_first_port_word():
    s = v7_atom_in_the_second_port_word()
    run = with_lists(s)
    i = s.meta["running"]["names"].index("ns/a1-web")
    groups = run["aff_group"][run["aff_group_off"][i]:run["aff_group_off"][i + 1]]
    # every group is read by a pending pod and no port is used, so group g becomes bit g: a1-web's second group sits in word 1
    assert s.pod_affinity["n_groups"] > 64 and atoms_fit(s) and len(groups) == 2 and max(groups) >= 64


# ------------------------------------------------------------------------------------------------ random clusters
def _random(s, what):
    """every tier variant x action list, bit-exact against the status-following oracle -> (cycles, cycles that evicted a member)"""
    if s.pod_affinity is None:                                       # no PodGroup drew the spread
        return 0, 0
    run = with_lists(s)
    member = (run["flags"] & abi.KB_RUNNING_AFF_MEMBER) != 0
    cycles = hit = 0
    for tname, tr in tier_variants():
        for acts in LISTS:
            o, ev, order = follow_oracle.cycle(s, tr, acts, run)
            g, gev, gorder = util.emu_cycle(s, tr, acts, run, mode=1)
            compare(f"{what} {tname} {acts}", o, ev, order, g, gev, gorder, util.emu_states(g))
            cycles += 1
            hit += bool((gev & member).any())
    return cycles, hit


@pytest.mark.parametrize("seed", range(24))
def test_random_spread_clusters_with_members_running(seed):
    c, h = _random(aff_gen.evict_spread_cluster(seed, members_running=True), f"seed {seed}")
    if c == 0:
        pytest.skip("no PodGroup drew the spread")


def test_random_spread_clusters_evict_members():
    """the clusters above exercise the new path: members are evicted in a good share of the cycles"""
    cycles = hit = 0
    for seed in range(24):
        s = aff_gen.evict_spread_cluster(seed, members_running=True)
        if s.pod_affinity is None:
            continue
        run = with_lists(s)
        member = (run["flags"] & abi.KB_RUNNING_AFF_MEMBER) != 0
        for tname, tr in tier_variants():
            for acts in LISTS:
                g, gev, _ = util.emu_cycle(s, tr, acts, run, mode=1)
                cycles += 1
                hit += bool((gev & member).any())
    assert hit >= cycles // 10, (hit, cycles)


@pytest.mark.parametrize("seed", range(6))
def test_random_spread_clusters_with_many_groups(seed):
    """more than 64 groups: atoms past the first port word"""
    s = aff_gen_many.evict_spread_cluster(seed, members_running=True, n_apps=300, n_pod_groups=90, W=2)
    assert s.pod_affinity["n_groups"] > 64 and atoms_fit(s)
    _random(s, f"many seed {seed}")


def test_without_the_lists_an_evicted_member_still_withholds():
    withheld = 0
    for seed in range(8):
        s = aff_gen.evict_spread_cluster(seed, members_running=True)
        try:
            util.emu_cycle(s, PluginConf.default(), LISTS[0], s.meta["running"], mode=1)
        except RuntimeError as ex:
            assert "withheld" in str(ex)
            withheld += 1
            util.emu_cycle(s, PluginConf.default(), LISTS[0], with_lists(s), mode=1)
    assert withheld > 0


@pytest.mark.parametrize("seed", range(6))
def test_the_status_following_oracle_agrees_where_no_member_is_evicted(seed):
    """the oracle variant changes nothing but the listing of evicted Running pods: without members running it equals the oracle"""
    s = aff_gen.evict_spread_cluster(seed, members_running=False)
    for tname, tr in tier_variants():
        for acts in LISTS:
            o, ev, order = kbo.cycle(s, tr, actions=acts, running=s.meta["running"])
            f, fev, forder = follow_oracle.cycle(s, tr, acts, s.meta["running"])
            compare(f"seed {seed} {tname} {acts}", o, ev, order, f, fev, forder)
            np.testing.assert_array_equal(o.node_ports, f.node_ports)


# ------------------------------------------------------------------------------------------------ refusals
def _rc(s, run):
    try:
        util.emu_cycle(s, PluginConf.default(), ("reclaim",), run, mode=1)
        return abi.KB_OK, ""
    except RuntimeError as ex:
        m = str(ex)
        return int(m.split("rc=")[1].split(":")[0]), m


def test_refusals():
    s = v2_one_of_two_members_evicted()
    run = with_lists(s)
    assert _rc(s, run)[0] == abi.KB_OK
    off, grp = np.array(run["aff_group_off"]), np.array(run["aff_group"])
    assert off[-1] > 0
    i = int(np.nonzero(np.diff(off))[0][0])
    # offsets that go backwards
    o = off.copy(); o[i + 1] = 0 if i + 2 < len(o) else o[i + 1]; o[i] = off[-1]
    rc, msg = _rc(s, dict(run, aff_group_off=o))
    assert rc == abi.KB_E_BADARG and "not monotone" in msg, msg
    # entries without the list
    r = dict(run); r.pop("aff_group")
    rc, msg = _rc(s, r)
    assert rc == abi.KB_E_BADARG and "NULL" in msg, msg
    # a group the session does not have
    g = grp.copy(); g[0] = s.pod_affinity["n_groups"]
    rc, msg = _rc(s, dict(run, aff_group=g))
    assert rc == abi.KB_E_BADARG and "names group" in msg, msg
    # more listed members in one domain than group_count0 holds there
    t = copy.copy(s)
    pa = dict(s.pod_affinity)
    c = np.array(pa["group_count0"]); c[c > 0] -= 1
    pa["group_count0"] = c
    t.pod_affinity = pa
    t.invalidate()
    rc, msg = _rc(t, run)
    assert rc == abi.KB_E_BADARG and "group_count0" in msg, msg


def test_builder_keeps_the_running_table_and_lists_every_member():
    s = v2_one_of_two_members_evicted()
    run, lists = s.meta["running"], s.meta["running_aff_groups"]
    assert "aff_group_off" not in run and "aff_group" not in run
    member = (run["flags"] & abi.KB_RUNNING_AFF_MEMBER) != 0
    has = np.diff(lists["aff_group_off"]) > 0
    assert (member == has).all()


def test_synth_members_match_the_spread_groups():
    s, _ = synth.make("c1")
    synth.add_host_spread(s, 0.5)
    run = synth.running_of(s, 0.3)
    c0 = np.array(s.pod_affinity["group_count0"]).copy()
    lists = synth.add_running_members(s, run, 0.2)
    member = (run["flags"] & abi.KB_RUNNING_AFF_MEMBER) != 0
    assert member.sum() == s.meta["member_tasks"] > 0
    assert (np.diff(lists["aff_group_off"])[member] == 2).all() and (np.diff(lists["aff_group_off"])[~member] == 0).all()
    assert int((np.array(s.pod_affinity["group_count0"]) - c0).sum()) == 2 * int(member.sum())
