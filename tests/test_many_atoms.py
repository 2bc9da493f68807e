"""Sessions with more than 256 label, taint or host-port atoms (W = 5..16 mask words, KB_MAX_W) against the oracle.

The engine runs such sessions on the kernels' wide-atom instances (class records of KB_MAX_W words).  CPU: the same algorithm run
by the emulation built with wide-atom class records (tests/emu_wide_atoms: tests/emu/kb_emu.cpp with KB_CLASS_W = KB_MAX_W) in
launch modes 0 / 1 / 5, on seeded synthetic sessions whose deciding atoms sit in the last word of each family, a per-team cluster
built from objects, and hand-computed cases decided by the atom at bit 1023.  The GPU twin is test_gpu_many_atoms.py."""
from __future__ import annotations

import contextlib
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from kube_batch_b200 import abi, builder as B, synth
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import util
from test_evict_parity import compare, tier_variants

_HERE = os.path.dirname(os.path.abspath(__file__))
FULL_LIST = ("reclaim", "allocate", "backfill", "preempt")            # config/kube-batch-conf.yaml:1
ACTION_LISTS = (("allocate",), ("allocate", "backfill"), FULL_LIST)
EMU_MODES = (0, 1, 5)                                                 # overlap, plain, persistent pipeline (falls back past W = 2)
TEAMS = 300
_lib = None


def atoms_lib():
    global _lib
    if _lib is None:
        d = os.path.join(_HERE, "emu_wide_atoms")
        with open(os.path.join(d, ".build.lock"), "w") as lk:
            import fcntl
            fcntl.flock(lk, fcntl.LOCK_EX)
            subprocess.check_call(["make", "-C", d, "-s"])
        _lib = C.CDLL(os.path.join(d, "libkbemu_wide_atoms.so"))
        _lib.kbemu_last_error.restype = C.c_char_p
    return _lib


@contextlib.contextmanager
def atoms_emulation():
    """util's emulation helpers, run by the emulation with wide-atom class records"""
    saved = util._emu
    util._emu = atoms_lib()
    try:
        yield
    finally:
        util._emu = saved


def check_cycle(s, tiers, acts, running, what, modes=EMU_MODES, oracle=kbo.cycle):
    o, ev, order = oracle(s, tiers, actions=acts, running=running)
    with atoms_emulation():
        for mode in modes:
            g, gev, gorder = util.emu_cycle(s, tiers, acts, running, mode=mode)
            compare(f"{what} mode {mode}", o, ev, order, g, gev, gorder, util.emu_states(g))
            util.assert_same_decisions(o.decisions, g.decisions, f"{what} mode {mode}")
    return o, ev, order


# ------------------------------------------------------------------------------------------------ synthetic sessions
HI = np.uint64(1) << np.uint64(63)


HI2 = np.uint64(1) << np.uint64(62)


def deepen(s, seed: int, pref: bool = False):
    """Moves deciding atoms into bit 63 of the last word of each family: a nodeSelector atom on half of the nodes that a sixth of
    the jobs require, a required node-affinity term on it, a NoSchedule taint on a tenth of the nodes that only a quarter of the
    jobs tolerate, and a host port some jobs own (and conflict on) that a few nodes already hold.  synth puts its own zone / ssd /
    taint atoms in words 0 and W - 1.  pref: a third of the jobs without a selector or required term (so that most nodes are
    feasible for them) also prefer bit 63 (weight 50) and bit 62 (weight 10, a third of the nodes) of the last label word."""
    rng = np.random.default_rng(9100 + seed)
    W, N, T = s.W, s.N, s.T
    off = s.job_task_off.astype(np.int64)
    tj = np.repeat(np.arange(s.J), np.diff(off))
    lab = rng.random(N) < 0.5
    s.node_labels[W - 1] |= np.where(lab, HI, np.uint64(0))
    s.node_taints[W - 1] |= np.where(rng.random(N) < 0.1, HI, np.uint64(0))
    s.node_ports[W - 1] |= np.where(rng.random(N) < 0.05, HI, np.uint64(0))
    u = rng.random(s.J)[tj]
    sel = u < 0.16
    s.task_sel_req[W - 1] |= np.where(sel, HI, np.uint64(0))
    s.task_tol[W - 1] |= np.where(rng.random(s.J)[tj] < 0.25, HI, np.uint64(0))
    port = (u >= 0.16) & (u < 0.2)
    s.task_port_own[W - 1] |= np.where(port, HI, np.uint64(0))
    s.task_port_conflict[W - 1] |= np.where(port, HI, np.uint64(0))
    # required node affinity (label at bit 63 of the last word) on a few jobs without other terms
    na = (u >= 0.2) & (u < 0.26) & (s.task_n_aff_terms[:T] == 0)
    s.task_n_aff_terms[:T] = np.where(na, 1, s.task_n_aff_terms[:T])
    s.task_aff_terms[0, W - 1] |= np.where(na, HI, np.uint64(0))
    if pref:
        s.node_labels[W - 1] |= np.where(rng.random(N) < 0.33, HI2, np.uint64(0))
        pt = np.nonzero((rng.random(s.J)[tj] < 0.33) & ~sel & ~na & (s.task_n_aff_terms[:T] == 0))[0]
        s.task_flags[pt] |= abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY
        s.task_n_pref_terms[pt] = 2
        s.task_pref_terms[0, W - 1, pt] = HI
        s.task_pref_weights[0, pt] = 50
        s.task_pref_terms[1, W - 1, pt] = HI2
        s.task_pref_weights[1, pt] = 10
    return s


def without_pref(s):
    """the same session without its preferred terms"""
    import copy
    s2 = copy.deepcopy(s)
    s2.task_flags[:] &= ~np.uint32(abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY)
    s2.task_n_pref_terms[:] = 0
    s2.task_pref_terms[:] = 0
    s2.task_pref_weights[:] = 0
    return s2


def pref_decides(s, run):
    """(placements, evictions) the preferred terms change: kb_allocate's nodes, and the victims of the shipped list"""
    conf = PluginConf.default()
    bare = without_pref(s)
    placed = int((kbo.allocate(s, conf).decisions["node"] != kbo.allocate(bare, conf).decisions["node"]).sum())
    evicted = 0
    for _, tiers in tier_variants():
        _, ev, order = kbo.cycle(s, tiers, actions=FULL_LIST, running=run)
        _, ev2, order2 = kbo.cycle(bare, tiers, actions=FULL_LIST, running=run)
        evicted += int((ev != ev2).sum() + (order != order2).sum())
    return placed, evicted


def synthetic(W, seed, pref):
    return deepen(synth.random_session(seed, tasks=300, jobs=40, nodes=40, queues=2, oversub=3.0, W=W), seed, pref)


@pytest.mark.parametrize("pref", [False, True], ids=["required", "preferred"])
@pytest.mark.parametrize("W", [5, 8, 16])
@pytest.mark.parametrize("seed", range(2))
def test_synthetic_sessions_on_the_emulation(W, seed, pref):
    s = synthetic(W, seed, pref)
    run = synth.running_of(s, 0.8, seed=seed + 1)
    evictions = 0
    for tname, tiers in tier_variants():
        for acts in ACTION_LISTS:
            o, ev, _ = check_cycle(s, tiers, acts, run, f"W {W} seed {seed} {tname} {acts}")
            evictions += int(ev.sum())
    assert s.W == W and evictions > 0
    # the last word decides: some task with the selector atom is placed, and only on a node that carries it
    o = kbo.allocate(s, PluginConf.default())
    sel = (s.task_sel_req[W - 1] & HI) != 0
    placed = sel & (o.decisions["node"] >= 0)
    assert placed.any()
    assert np.all((s.node_labels[W - 1][o.decisions["node"][placed]] & HI) != 0)
    if pref:                                                           # the preferred terms in the last word move placements and victims
        moved, evicted = pref_decides(s, run)
        assert moved > 0 and evicted > 0, (moved, evicted)


# ------------------------------------------------------------------------------------------------ objects: one pool per team
G = 1e9


def team_cluster(teams: int = TEAMS, selectors: str = "label", running: bool = False) -> B.SessionBuilder:
    """One queue, one labelled (team=<t>) and tainted (dedicated=<t>:NoSchedule) node per team, and per team a PodGroup of two
    pods with the matching nodeSelector (or required / preferred node affinity: In, NotIn, Exists, Gt, Lt) and toleration.  Each
    node fits one pod, so the second pod of a team stays Pending.  running: every team's node already runs a low-priority pod of
    the team's queue (preempt picks it) and a shared "batch" queue holds pods that tolerate every taint on a few teams' nodes
    (reclaim picks those)."""
    b = B.SessionBuilder()
    for t in range(teams):
        b.add_queue(B.Queue(f"q{t:03d}", 1))
    b.add_queue(B.Queue("batch", 1))
    for t in range(teams):
        name = f"t{t:03d}"
        b.add_node(B.Node(f"n{t:03d}", {"cpu": 4, "memory": 8 * G, "pods": 110},
                          labels={"team": name, "rank": str(t)}, taints=[("dedicated", name, "NoSchedule")]))
    for t in range(teams):
        name = f"t{t:03d}"
        tol = [("dedicated", "Equal", name, "NoSchedule")]
        kw = {}
        if selectors == "label":
            kw["node_selector"] = {"team": name}
        else:
            form = t % 4
            if form == 0:
                kw["affinity_terms"] = [[("team", "In", [name])]]
            elif form == 1:
                kw["affinity_terms"] = [[("team", "Exists", []), ("rank", "Gt", [str(t - 1)]), ("rank", "Lt", [str(t + 1)])]]
            elif form == 2:
                kw["affinity_terms"] = [[("team", "In", [name]), ("rank", "NotIn", [str(t + 1)])]]
            else:
                kw["node_selector"] = {"team": name}
            kw["preferred_terms"] = [(5, [("team", "In", [name])])]
        b.add_pod_group(B.PodGroup("ns", f"g{t:03d}", f"q{t:03d}", min_member=1, priority=100))
        for k in range(2):
            b.add_pod(B.Pod("ns", f"p{t:03d}-{k}", requests={"cpu": 3, "memory": 1 * G}, group=f"g{t:03d}", tolerations=tol,
                            priority=100, **kw))
        if running:
            b.add_pod_group(B.PodGroup("ns", f"low{t:03d}", f"q{t:03d}", min_member=1, priority=0))
            b.add_pod(B.Pod("ns", f"low{t:03d}", f"n{t:03d}", "Running", {"cpu": 2, "memory": 1 * G}, group=f"low{t:03d}",
                            tolerations=tol, priority=0))
    if running:
        b.add_pod_group(B.PodGroup("ns", "batch", "batch", min_member=1))
        for t in range(0, teams, 7):
            b.add_pod(B.Pod("ns", f"batch{t:03d}", f"n{t:03d}", "Running", {"cpu": 1, "memory": 1 * G}, group="batch",
                            tolerations=[("", "Exists", "", "")]))
    return b


@pytest.mark.parametrize("selectors", ["label", "affinity"])
def test_per_team_cluster_on_the_emulation(selectors):
    b = team_cluster(selectors=selectors)
    s = b.flatten()
    assert 5 <= s.W <= abi.KB_MAX_W, s.W                              # 300 team labels and 300 taints: at least 5 words
    o = None
    for acts in (("allocate",), ("allocate", "backfill")):
        o, _, _ = check_cycle(s, PluginConf.default(), acts, s.meta["running"], f"teams {selectors} {acts}")
    # every team's first pod lands on its own node, teams 256.. through atoms in word 4
    nodes = o.decisions["node"]
    placed = {t: int(n) for t, n in enumerate(nodes) if n >= 0}
    names, tnames = s.meta["nodes"], s.meta["tasks"]
    assert len(placed) == TEAMS
    for t, n in placed.items():
        assert names[n][1:] == tnames[t].split("/")[1][1:4], (tnames[t], names[n])
    assert any(int(tnames[t].split("/")[1][1:4]) >= 256 for t in placed)


def test_per_team_cluster_with_running_pods_on_the_emulation():
    b = team_cluster(running=True)
    s = b.flatten()
    assert s.W == 5
    run = s.meta["running"]
    evicted_hi = 0
    for tname, tiers in tier_variants():
        o, ev, order = check_cycle(s, tiers, FULL_LIST, run, f"teams running {tname}", modes=(0, 1))
        names = [run["names"][i] for i in np.nonzero(ev)[0]]
        evicted_hi += sum(1 for nm in names if nm.split("/")[1].startswith("low") and int(nm.split("/")[1][3:]) >= 256)
    assert evicted_hi > 0                                              # preempt picked victims on nodes whose taint sits in word 4


def test_the_cpp_mirror_flattens_the_per_team_cluster_like_builder(tmp_path):
    """kbhost.hpp's Flatten (tests/host affinity_run --flat; no GPU) on the same objects: the same node-affinity relations"""
    import test_host_cpp_affinity as HA
    HA._build()
    for selectors in ("label", "affinity"):
        HA.check_flat(tmp_path, team_cluster(selectors=selectors, running=True))


# ------------------------------------------------------------------------------------------------ host-level anti-affinity past word 4
HOSTNAME = "kubernetes.io/hostname"
PORTS = 300


def anti_affinity_cluster(anti: bool = True) -> B.SessionBuilder:
    """300 pods on a tainted port pool hold 300 distinct host ports (port atoms 0..299), so the hostname anti-affinity groups of apps a
    and b become atoms 300 and 301: port-word bits in word 4.  Every node carries its hostname label.
      n00 runs a low-priority member of app a, n01 a low-priority non-member of the same size; each node fits one such pod.  A
      pending high-priority pod of app a (anti-affine to app a) of that size fits nowhere, so preempt evicts: the non-member on
      n01 — without the anti-affinity the member on n00 (the lower node of two equal ones).
      n02 runs a small member of app b, n03 a bigger non-member.  A pending pod of app b goes to n03 — without the anti-affinity
      to n02, the less requested node.
    anti=False: the same pods without their anti-affinity terms."""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_queue(B.Queue("qp", 1))
    for i in range(4):
        b.add_node(B.Node(f"n{i:02d}", {"cpu": 4, "memory": 8 * G, "pods": 110}, labels={HOSTNAME: f"n{i:02d}"}))
    b.add_node(B.Node("zports", {"cpu": 1000, "memory": 1000 * G, "pods": 1000}, labels={HOSTNAME: "zports", "pool": "ports"},
                      taints=[("pool", "ports", "NoSchedule")]))
    b.add_pod_group(B.PodGroup("ns", "ports", "qp", min_member=1))
    for i in range(PORTS):
        b.add_pod(B.Pod("ns", f"port{i:03d}", requests={"cpu": 1, "memory": G}, group="ports", node_selector={"pool": "ports"},
                        host_ports=[("", "TCP", 20000 + i)], priority=0, tolerations=[("pool", "Equal", "ports", "NoSchedule")]))

    def aa(app):
        return dict(labels={"app": app},
                    pod_anti_affinity=B.PodAffinity(required=[B.PodAffinityTerm(HOSTNAME, match_labels={"app": app})]) if anti else None)
    b.add_pod_group(B.PodGroup("ns", "low", "q", min_member=1, priority=0))
    b.add_pod(B.Pod("ns", "low-a", "n00", "Running", {"cpu": 3, "memory": G}, group="low", priority=0, **aa("a")))
    b.add_pod(B.Pod("ns", "low-x", "n01", "Running", {"cpu": 3, "memory": G}, group="low", priority=0))
    b.add_pod(B.Pod("ns", "run-b", "n02", "Running", {"cpu": 1.5, "memory": G}, group="low", priority=0, **aa("b")))
    b.add_pod(B.Pod("ns", "run-y", "n03", "Running", {"cpu": 2.5, "memory": G}, group="low", priority=0))
    b.add_pod_group(B.PodGroup("ns", "hi", "q", min_member=1, priority=100))
    b.add_pod(B.Pod("ns", "hi-a", requests={"cpu": 3, "memory": G}, group="hi", priority=100, **aa("a")))
    b.add_pod_group(B.PodGroup("ns", "web", "q", min_member=1, priority=50))
    b.add_pod(B.Pod("ns", "web-b", requests={"cpu": 1, "memory": G}, group="web", priority=50, **aa("b")))
    return b


def anti_affinity_outcome(s, decisions, ev):
    """(node of web-b, evicted Running pods) by name"""
    tasks, nodes, run = s.meta["tasks"], s.meta["nodes"], s.meta["running"]
    web = int(decisions["node"][tasks.index("ns/web-b")])
    return (nodes[web] if web >= 0 else None), sorted(run["names"][i] for i in np.nonzero(ev)[0])


def members_listed(s):
    """the Running table with builder.py's group lists merged in (an evicted member's atoms are cleared on its node)"""
    return dict(s.meta["running"], **s.meta["running_aff_groups"])


def test_host_level_anti_affinity_past_word_4_on_the_emulation():
    import follow_oracle
    s = anti_affinity_cluster().flatten()
    assert s.W == 5 and s.pod_affinity is not None
    run = members_listed(s)
    for acts in (("allocate",), FULL_LIST):
        o, ev, _ = check_cycle(s, PluginConf.default(), acts, run, f"anti-affinity {acts}", oracle=follow_oracle.cycle)
    # the group atoms (bits 300, 301) decide: web-b avoids n02, preempt evicts the non-member on n01
    assert anti_affinity_outcome(s, o.decisions, ev) == ("n03", ["ns/low-x"])
    bare = anti_affinity_cluster(anti=False).flatten()
    o2, ev2, _ = kbo.cycle(bare, PluginConf.default(), actions=FULL_LIST, running=bare.meta["running"])
    assert anti_affinity_outcome(bare, o2.decisions, ev2) == ("n02", ["ns/low-a"])
    evicted_member = False
    for tname, tiers in tier_variants():
        _, ev, _ = check_cycle(s, tiers, FULL_LIST, run, f"anti-affinity {tname}", modes=(0, 1), oracle=follow_oracle.cycle)
        evicted_member |= "ns/low-a" in anti_affinity_outcome(s, o.decisions, ev)[1]
    assert evicted_member                                              # some variant's reclaim evicts the member of app a


# ------------------------------------------------------------------------------------------------ hand-computed cases
def _two_nodes(family: str):
    """Two empty nodes, one pending pod, W = 16; the only difference between the nodes is the atom at bit 1023 of `family`.
    Node 0 wins every tie (lowest index), so the pod lands on node 1 only if bit 1023 is read."""
    s = synth.random_session(0, tasks=1, jobs=1, nodes=2, W=16)
    for a in (s.node_labels, s.node_taints, s.node_ports, s.task_sel_req, s.task_tol, s.task_port_own, s.task_port_conflict):
        a[:] = 0
    s.task_aff_terms[:] = 0
    s.task_n_aff_terms[:] = 0
    s.node_flags[:] = 0
    s.node_idle[:] = s.node_allocatable[:, :1]
    s.node_allocatable[:] = s.node_allocatable[:, :1]
    s.node_releasing[:] = 0
    s.node_used[:] = 0
    s.node_pods[:] = 0
    s.node_nz_cpu[:] = 0
    s.node_nz_mem[:] = 0
    s.node_alloc_cpu[:] = s.node_alloc_cpu[0]
    s.node_alloc_mem[:] = s.node_alloc_mem[0]
    s.node_alloc_present[:] = s.node_alloc_present[0]
    if family == "selector":
        s.node_labels[15, 1] = HI
        s.task_sel_req[15, 0] = HI
    elif family == "affinity":
        s.node_labels[15, 1] = HI
        s.task_n_aff_terms[0] = 1
        s.task_aff_terms[0, 15, 0] = HI
    elif family == "taint":
        s.node_taints[15, 0] = HI                                    # untolerated on node 0
    elif family == "port":
        s.node_ports[15, 0] = HI
        s.task_port_own[15, 0] = HI
        s.task_port_conflict[15, 0] = HI
    elif family == "preferred":                                       # both nodes feasible, node 1 preferred
        s.node_labels[15, 1] = HI
        s.task_flags[0] |= abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY
        s.task_n_pref_terms[0] = 1
        s.task_pref_terms[0, 15, 0] = HI
        s.task_pref_weights[0, 0] = 10
    return s


HAND = ["selector", "affinity", "taint", "port", "preferred"]


@pytest.mark.parametrize("family", HAND)
def test_hand_computed_cases_on_the_emulation(family):
    s = _two_nodes(family)
    o = kbo.allocate(s, PluginConf.default())
    assert int(o.decisions["node"][0]) == 1, o.decisions
    with atoms_emulation():
        for mode in EMU_MODES:
            util.assert_same_decisions(o.decisions, util.emu_allocate(s, PluginConf.default(), mode=mode).decisions, f"{family} mode {mode}")
    # without the atom the pod takes node 0: the atom decides
    for a in (s.node_labels, s.node_taints, s.node_ports, s.task_sel_req, s.task_port_own, s.task_port_conflict):
        a[15] = 0
    s.task_n_aff_terms[:] = 0
    assert int(kbo.allocate(s, PluginConf.default()).decisions["node"][0]) == 0


# ------------------------------------------------------------------------------------------------ refusals
def test_more_than_1024_atoms_are_refused():
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_node(B.Node("n", {"cpu": 4, "memory": 8 * G, "pods": 110}, taints=[("k", str(i), "NoSchedule") for i in range(1025)]))
    b.add_pod_group(B.PodGroup("ns", "g", "q", min_member=1))
    b.add_pod(B.Pod("ns", "p", requests={"cpu": 1, "memory": G}, group="g"))
    with pytest.raises(AssertionError, match=r"1025 label / taint / port atoms > 64 x KB_MAX_W \(16\)"):
        b.flatten()
    s = synth.random_session(1, tasks=40, jobs=6, nodes=8, W=16)
    cs, keep = s.to_c()
    cs.W = abi.KB_MAX_W + 1
    s.to_c = lambda: (cs, keep)
    with atoms_emulation(), pytest.raises(RuntimeError, match=r"rc=-1: R=3 / W=17 out of range .*1 <= W <= KB_MAX_W = 16"):
        util.emu_allocate(s, PluginConf.default())


def test_many_dimensions_with_many_atoms_are_refused():
    s = synth.random_session(1, tasks=40, jobs=6, nodes=8, R=9, W=5)
    with atoms_emulation(), pytest.raises(RuntimeError, match=r"R=9 resource dimensions with W=5 mask words: .*KB_NARROW_R \(8\).*KB_NARROW_W \(4\)"):
        util.emu_allocate(s, PluginConf.default())
    b = team_cluster(teams=260)
    b.nodes[0].allocatable.update({f"example.com/s{i}": 1.0 for i in range(7)})     # R = 9
    with pytest.raises(AssertionError, match=r"9 resource dimensions > KB_NARROW_R \(8\) with 260 atoms > 64 x KB_NARROW_W \(4\)"):
        b.flatten()


def test_the_cpp_mirror_refuses_many_dimensions_with_many_atoms(tmp_path):
    import test_host_cpp_affinity as HA
    HA._build()
    b = team_cluster(teams=260)
    b.nodes[0].allocatable.update({f"example.com/s{i}": 1.0 for i in range(7)})     # R = 9
    HA._refused(tmp_path, b, "9 resource dimensions > KB_NARROW_R (8) with 260 atoms > 64 x KB_NARROW_W (4)")


def test_the_narrow_emulation_refuses_wide_atom_sessions():
    """host code that reads the class table as 4-word records (tests/emu) is told so instead of misreading a wide-atom table"""
    s = synth.random_session(3, tasks=40, jobs=6, nodes=8, W=5)
    with pytest.raises(RuntimeError, match="class records of 4 mask words"):
        util.emu_allocate(s, PluginConf.default())


def _sharded_rank(rank, world, port, W, q):
    import util as U
    import test_many_atoms as M
    U._emu = M.atoms_lib()
    s = synth.random_session(2, tasks=60, jobs=8, nodes=300, W=W)
    try:
        out = U.emu_sharded_rank(rank, world, port, s, PluginConf.default())
        ref = kbo.allocate(s, PluginConf.default())
        U.assert_same_decisions(ref.decisions, out.decisions, f"W={W} rank {rank}")
        q.put((rank, "ok"))
    except Exception as e:                                                    # noqa: BLE001 — the message travels to the parent
        q.put((rank, str(e)))


@pytest.mark.parametrize("W", [4, 5])
def test_a_sharded_gloo_world_of_two(W):
    """A sharded node axis takes W <= 4 (the exchange's records); W = 5 is refused on every rank, naming the limit"""
    import multiprocessing as mp
    import socket
    sk = socket.socket()
    sk.bind(("127.0.0.1", 0))
    port = sk.getsockname()[1]
    sk.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_rank, args=(r, 2, port, W, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    for rank in range(2):
        if W <= 4:
            assert res[rank] == "ok", res
        else:
            assert "W=5 mask words with a sharded node axis (KB_ENGINE_SHARD)" in res[rank], res
            assert "KB_NARROW_W (4)" in res[rank], res
