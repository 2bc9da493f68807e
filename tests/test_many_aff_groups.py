"""More than 64 inter-pod affinity counter groups.  Groups 0..63 stay bits of kb_pod_affinity.task_forbid / task_contrib, groups
64 and above are per-task entries of task_xgroup (include/kbgpu.h); the host build resolves them into per-class lists (kb_build.h)
that aff_pred / aff_self_blocks / aff_commit walk after the masks (kb_aff.h).  The emulation of the device algorithm is checked
against the object-level oracle, which walks the raw pods and has no group limit."""
import copy
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from kube_batch_b200 import abi, builder as B, synth
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import aff_gen
import aff_gen_many
import util
import test_pod_affinity as tpa

HOST = tpa.HOST
FORBID, CONTRIB = abi.KB_XGROUP_FORBID, abi.KB_XGROUP_CONTRIB
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------- helpers: decode / re-encode the per-task group sets ----------------
def group_sets(pa, T):
    """-> per task (forbidden groups, joined groups), over every group of the session"""
    xo, xg = pa.get("task_xgroup_off"), pa.get("task_xgroup")
    out = []
    for t in range(T):
        f = {g for g in range(64) if (int(pa["task_forbid"][t]) >> g) & 1}
        c = {g for g in range(64) if (int(pa["task_contrib"][t]) >> g) & 1}
        if xo is not None:
            for e in xg[int(xo[t]):int(xo[t + 1])]:
                e = int(e)
                if e & FORBID:
                    f.add(e >> 2)
                if e & CONTRIB:
                    c.add(e >> 2)
        out.append((f, c))
    return out


def encode(pa, sets):
    """writes the masks (groups < 64) and the lists (groups >= 64, ascending) of `sets` into pa"""
    fm, cm, off, lst = [], [], [0], []
    for f, c in sets:
        fm.append(sum(1 << g for g in f if g < 64))
        cm.append(sum(1 << g for g in c if g < 64))
        for g in sorted(x for x in f | c if x >= 64):
            lst.append((g << 2) | (FORBID if g in f else 0) | (CONTRIB if g in c else 0))
        off.append(len(lst))
    pa["task_forbid"] = np.array(fm or [0], dtype=np.uint64)
    pa["task_contrib"] = np.array(cm or [0], dtype=np.uint64)
    pa["task_xgroup_off"] = np.array(off, dtype=np.uint32)
    pa["task_xgroup"] = np.array(lst or [0], dtype=np.uint32)


def relabel(snap, perm):
    """the same session with group g renamed perm[g]: masks, lists, key sets, counters, totals and needed groups move with it"""
    pa = dict(snap.pod_affinity)
    NG, T = int(pa["n_groups"]), snap.T
    dom = [int(pa["keyset_domains"][int(pa["group_keyset"][g])]) for g in range(NG)]
    off = np.concatenate([[0], np.cumsum(dom)]).astype(np.int64)
    inv = np.argsort(perm)                                  # inv[new id] = old id
    pa["group_keyset"] = np.array([pa["group_keyset"][inv[h]] for h in range(NG)], dtype=np.uint32)
    pa["group_total0"] = np.array([pa["group_total0"][inv[h]] for h in range(NG)], dtype=np.int32)
    blocks = [np.asarray(pa["group_count0"][off[inv[h]]:off[inv[h] + 1]]) for h in range(NG)]
    pa["group_count0"] = np.concatenate(blocks).astype(np.int32) if off[NG] else np.zeros(1, dtype=np.int32)
    need = np.array(pa["task_need"], dtype=np.int32)
    need[:T] = [perm[n] if n >= 0 else -1 for n in need[:T]]
    pa["task_need"] = need
    encode(pa, [({perm[g] for g in f}, {perm[g] for g in c}) for f, c in group_sets(snap.pod_affinity, T)])
    r = copy.copy(snap)
    r.pod_affinity = pa
    r.invalidate()
    return r


def forty_apps(replica_node: str):
    """40 "one replica per host" apps = 80 counter groups on 2 nodes.  n1 is the busier node (a filler pod), so every placement
    prefers n0; app a39's Running replica sits on `replica_node` and carries the label but no term: it is a member of one group only,
    the one of a39's own term list (group 79)."""
    sb = B.SessionBuilder()
    sb.add_queue(B.Queue("q1"))
    for i in range(2):
        sb.add_node(B.build_node(f"n{i}", B.build_resource_list("64", "128Gi"), labels={HOST: f"n{i}"}, pods=110))
    sb.add_pod_group(B.PodGroup("ns", "pg1", "q1", min_member=1))
    sb.add_pod_group(B.PodGroup("ns", "run", "q1", min_member=1))
    sb.add_pod(tpa.pod("filler", {"app": "filler"}, node="n1", phase="Running", group="run", cpu="8"))
    sb.add_pod(tpa.pod("a39-run", {"app": "a39"}, node=replica_node, phase="Running", group="run"))
    for k in range(40):
        p = tpa.pod(f"a{k}", {"app": f"a{k}"}, creation=0 if k == 39 else 1 + k)
        p.pod_anti_affinity = B.PodAffinity(required=[tpa.term(HOST, app=f"a{k}")])
        sb.add_pod(p)
    return sb.flatten()


def many_owners(n_owners=200, n_nodes=300):
    """n_owners Running pods on nodes 0 .. n_owners-1, each with its own required anti-affinity term {app NotIn [x<k>], hostname}
    that every pending pod matches: the pending class is forbidden by n_owners groups (136 of them >= 64, more than the scan stages
    in shared memory).  The other nodes carry a filler pod, so without the terms the pending pods would prefer the owners' nodes."""
    sb = B.SessionBuilder()
    sb.add_queue(B.Queue("q1"))
    for i in range(n_nodes):
        sb.add_node(B.build_node(f"n{i:03d}", B.build_resource_list("8", "16Gi"), labels={HOST: f"n{i:03d}"}, pods=110))
    sb.add_pod_group(B.PodGroup("ns", "pg1", "q1", min_member=1))
    sb.add_pod_group(B.PodGroup("ns", "run", "q1", min_member=1))
    for k in range(n_nodes):
        if k < n_owners:
            p = tpa.pod(f"o{k}", {"app": f"o{k}"}, node=f"n{k:03d}", phase="Running", group="run", cpu="100m")
            p.pod_anti_affinity = B.PodAffinity(required=[B.PodAffinityTerm(HOST, match_expressions=[("app", "NotIn", [f"x{k}"])])])
        else:
            p = tpa.pod(f"f{k}", {"app": "filler"}, node=f"n{k:03d}", phase="Running", group="run", cpu="4")
        sb.add_pod(p)
    for i in range(6):
        sb.add_pod(tpa.pod(f"v{i}", {"app": "v"}, creation=i))
    return sb.flatten()


def check(snap, conf, what, actions=3, modes=(1,)):
    o = kbo.allocate(snap, conf, actions=actions)
    for mode in modes:
        e = util.emu_allocate(snap, conf, actions=actions, mode=mode)
        util.assert_same_decisions(o.decisions, e.decisions, f"{what} mode {mode}")
        st = util.emu_states(e)
        util.assert_same_state(o, st[0], st[1], f"{what} mode {mode}")
    return o


def atoms_fit(snap, conf_predicates=True):
    """kb_build.h's rule for a host-level session: every group a task reads or joins becomes a spare bit of the port words"""
    used = set()
    if conf_predicates:
        for f, c in group_sets(snap.pod_affinity, snap.T):
            used |= f | c
    acc = [int(np.bitwise_or.reduce(np.concatenate([np.asarray(snap.node_ports[w]).ravel(), np.asarray(snap.task_port_own[w]).ravel(),
                                                    np.asarray(snap.task_port_conflict[w]).ravel(), [0]]).astype(np.uint64)))
           for w in range(snap.W)]
    hb = max([w * 64 + a.bit_length() - 1 for w, a in enumerate(acc) if a] or [-1])
    return hb + 1 + len(used) <= 64 * snap.W


# ---------------- 1. a hand-computed vector where only a group >= 64 decides ----------------
@pytest.mark.parametrize("replica_node,expect", [("n0", 1), ("n1", 0)])
def test_only_a_group_above_63_keeps_a39_off_its_replicas_node(replica_node, expect):
    snap = forty_apps(replica_node)
    pa = snap.pod_affinity
    assert pa["n_groups"] == 80 and pa["task_xgroup_off"] is not None
    assert np.nonzero(pa["group_total0"])[0].tolist() == [79]      # the replica is a member of group 79 only
    t39 = snap.meta["tasks"].index("ns/a39")
    f, c = group_sets(pa, snap.T)[t39]
    assert 79 in f and 79 in c and all(int(pa["group_total0"][g]) == 0 for g in f if g != 79)
    for ci, conf in enumerate(tpa.AFF_CONFS):
        o = check(snap, conf, f"replica on {replica_node} conf {ci}", actions=1, modes=(0, 1))
        node = int(o.decisions["node"][t39])
        if ci == 3:                                                  # no predicates plugin: step 10 is never evaluated
            continue
        assert o.decisions["kind"][t39] == abi.KB_KIND_ALLOCATED and node != int(replica_node[1:])
        if ci == 0:
            assert node == expect                                    # n0 wins on resources unless the replica sits there


def test_a_class_forbidden_by_two_hundred_groups():
    """200 forbidden groups, 136 of them in the list: the pending pods avoid every owner's node"""
    snap = many_owners()
    assert snap.pod_affinity["n_groups"] == 200 and int(snap.pod_affinity["task_xgroup_off"][1]) == 136
    for ci, conf in enumerate(tpa.AFF_CONFS[:3]):
        o = check(snap, conf, f"conf {ci}", actions=3, modes=(0, 1))
        assert (o.decisions["kind"] == abi.KB_KIND_ALLOCATED).all() and (o.decisions["node"] >= 200).all()


# ---------------- 2. relabelling across the 64 boundary ----------------
def _relabel_cases():
    yield "forty apps", forty_apps("n0")
    for seed in range(3):
        s = aff_gen_many.random_affinity_session(50 + seed, n_nodes=10 + seed, n_groups=120, n_apps=48).flatten()
        yield f"random {seed}", s


@pytest.mark.parametrize("case", range(4))
def test_relabelling_groups_across_the_boundary_changes_nothing(case):
    """The mask path and the list path mean the same thing: renaming the groups (reversed ids, then a random permutation) moves
    groups < 64 into the lists and groups >= 64 into the masks; decisions and node / job state stay those of the oracle."""
    what, snap = list(_relabel_cases())[case]
    NG = int(snap.pod_affinity["n_groups"])
    assert NG > 64
    rng = np.random.default_rng(case)
    for conf_i, conf in enumerate(tpa.AFF_CONFS):
        o = kbo.allocate(snap, conf, actions=3)
        base = util.emu_allocate(snap, conf, actions=3, mode=1)
        util.assert_same_decisions(o.decisions, base.decisions, f"{what} conf {conf_i}")
        for pname, perm in (("reversed", np.arange(NG)[::-1].copy()), ("random", rng.permutation(NG))):
            r = relabel(snap, perm)
            moved = sum(1 for g in range(NG) if (g < 64) != (perm[g] < 64))
            assert moved > 0
            e = util.emu_allocate(r, conf, actions=3, mode=1)
            util.assert_same_decisions(base.decisions, e.decisions, f"{what} conf {conf_i} {pname}")
            st = util.emu_states(e)
            util.assert_same_state(o, st[0], st[1], f"{what} conf {conf_i} {pname}")


# ---------------- 3. random sessions with 65-300 groups ----------------
@pytest.mark.parametrize("seed", range(16))
def test_random_sessions_with_many_groups_match_the_oracle(seed):
    sb = aff_gen_many.random_affinity_session(seed, n_nodes=6 + seed % 13, n_groups=100 + 10 * (seed % 5), n_apps=40 + 4 * (seed % 6),
                                         besteffort=seed % 4 == 3)
    snap = sb.flatten()
    assert 65 <= snap.pod_affinity["n_groups"] <= 300, snap.pod_affinity["n_groups"]
    assert int(snap.pod_affinity["task_xgroup_off"][-1]) > 0
    for ci, conf in enumerate(tpa.AFF_CONFS):
        for actions in (1, 3):
            check(snap, conf, f"seed {seed} conf {ci} actions {actions}", actions=actions, modes=(0, 1, 5))


# ---------------- 4. host-level spread with more than 64 groups ----------------
@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("fit", [True, False])
def test_host_spread_with_many_groups_as_atoms_or_counters(seed, fit):
    """Groups that fit the spare bits of the port words become atoms (cycle_kernel); the others stay on the counter path.  Both
    equal the oracle in every launch mode, and the counter path (KB_AFF_ATOMS=0) agrees."""
    n_apps, n_pg = (40, 80) if fit else (120, 150)
    snap = aff_gen_many.host_spread_session(900 + seed, n_nodes=6 + seed % 11, n_groups=n_pg, pipe_geometry=True, ports=seed % 3 == 0,
                                       n_apps=n_apps).flatten(W=2)
    NG = int(snap.pod_affinity["n_groups"])
    if fit and NG <= 64:
        pytest.skip("fewer than 65 groups drawn")
    assert NG > 64 and atoms_fit(snap) == fit
    for ci, conf in enumerate((PluginConf.default(), PluginConf.from_names([["gang"], ["predicates"]]))):
        o = check(snap, conf, f"seed {seed} conf {ci}", actions=3, modes=(0, 1, 5))
        os.environ["KB_AFF_ATOMS"] = "0"
        try:
            e = util.emu_allocate(snap, conf, actions=3, mode=1)
        finally:
            os.environ.pop("KB_AFF_ATOMS", None)
        util.assert_same_decisions(o.decisions, e.decisions, f"seed {seed} conf {ci} counter path")


@pytest.mark.parametrize("seed", range(10))
def test_shipped_action_list_on_spread_clusters_with_many_groups(seed):
    """reclaim, allocate, backfill, preempt on clusters whose pending pods spread ~50 labels (more than 64 groups, atoms of two port
    words): no placed pod is a member, so the atoms stay exact through the evictions; with members running, evicting one withholds
    the outcome."""
    from test_evict_parity import compare, tier_variants
    for members in (False, True):
        s = aff_gen_many.evict_spread_cluster(seed, members_running=members, n_apps=300, n_pod_groups=90, W=2)
        assert s.pod_affinity is not None and s.pod_affinity["n_groups"] > 64 and atoms_fit(s)
        member = (s.meta["running"]["flags"] & abi.KB_RUNNING_AFF_MEMBER) != 0
        assert members or not member.any()
        for tname, tiers in tier_variants():
            for acts in (("reclaim", "allocate", "backfill", "preempt"), ("allocate", "preempt")):
                o, ev, order = kbo.cycle(s, tiers, actions=acts, running=s.meta["running"])
                try:
                    g, gev, gorder = util.emu_cycle(s, tiers, acts, s.meta["running"], mode=1)
                except RuntimeError as ex:
                    assert members and "withheld" in str(ex), str(ex)
                    continue
                compare(f"seed {seed} members {members} {tname} {acts}", o, ev, order, g, gev, gorder, util.emu_states(g))
                assert not (ev & member).any()


# ---------------- 5. refusals ----------------
def build_rc(snap, conf=None):
    """kb_session_load's host build (kb_build.h) on the emulation -> (status, message)"""
    L = C.CDLL(util.emu_lib()._name)
    L.kbemu_create2.restype = C.c_void_p
    L.kbemu_create2.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    L.kbemu_reload.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    L.kbemu_destroy.argtypes = [C.c_void_p]
    L.kbemu_last_error.restype = C.c_char_p
    conf = conf or PluginConf.default()
    base = forty_apps("n0")
    cb, k0 = base.to_c()
    cc, k1 = conf.to_c()
    h = L.kbemu_create2(C.addressof(cb), C.addressof(cc), 0, 1, 1)
    assert h
    try:
        cs, k2 = snap.to_c()
        rc = L.kbemu_reload(h, C.addressof(cs), C.addressof(cc), 1)
        return rc, L.kbemu_last_error().decode()
    finally:
        L.kbemu_destroy(h)


def _with(snap, **changes):
    """a shallow copy of snap whose kb_pod_affinity has `changes` (None drops the array: a NULL pointer)"""
    r = copy.copy(snap)
    r.pod_affinity = {k: v for k, v in dict(snap.pod_affinity, **changes).items() if v is not None}
    r.invalidate()
    return r


def test_refusals():
    snap = forty_apps("n0")
    assert build_rc(snap) == (abi.KB_OK, build_rc(snap)[1])
    pa = snap.pod_affinity
    xo, xg = np.array(pa["task_xgroup_off"]), np.array(pa["task_xgroup"])
    # more groups than KB_MAX_AFF_GROUPS: unsupported (the shim runs the Go actions)
    G = abi.KB_MAX_AFF_GROUPS + 1
    rc, msg = build_rc(_with(snap, n_groups=G, group_keyset=np.zeros(G, np.uint32), group_total0=np.zeros(G, np.int32),
                             group_count0=np.zeros(G * snap.N, np.int32)))
    assert rc == abi.KB_E_UNSUPPORTED_FEATURE and "counter groups" in msg, msg
    # entries that do not name a group >= 64 of the session
    for bad in ((5 << 2) | FORBID, (80 << 2) | FORBID, 70 << 2):
        x = xg.copy(); x[0] = bad
        rc, msg = build_rc(_with(snap, task_xgroup=x))
        assert rc == abi.KB_E_BADARG and "task_xgroup entry" in msg, msg
    # offsets that go backwards
    o = xo.copy(); i = int(np.nonzero(np.diff(o))[0][0]); o[i + 1] = o[i] - 1 if o[i] else 0; o[i] = o[i] + 1
    rc, msg = build_rc(_with(snap, task_xgroup_off=o))
    assert rc == abi.KB_E_BADARG and "not monotone" in msg, msg
    # offsets that name entries, no entries
    rc, msg = build_rc(_with(snap, task_xgroup=None))
    assert rc == abi.KB_E_BADARG and "NULL" in msg, msg
    # a mask bit beyond n_groups is still refused for small sessions
    small = tpa.cluster(2)
    p = tpa.pod("p0", {"app": "web"})
    p.pod_anti_affinity = B.PodAffinity(required=[tpa.term(HOST, app="web")])
    small.add_pod(p)
    s = small.flatten()
    rc, msg = build_rc(_with(s, task_forbid=np.array([1 << 7], dtype=np.uint64)))
    assert rc == abi.KB_E_BADARG, msg


# ---------------- layout ----------------
def test_kb_pod_affinity_ctypes_mirror_has_the_c_size():
    src = '#include <stdio.h>\n#include "kbgpu.h"\nint main(void) { printf("%zu\\n", sizeof(kb_pod_affinity)); return 0; }\n'
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "s.c")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), c, "-o", os.path.join(d, "s")])
        assert int(subprocess.check_output([os.path.join(d, "s")])) == C.sizeof(abi.kb_pod_affinity)


def test_sessions_with_at_most_64_groups_carry_no_lists():
    s, _ = synth.make("c1")
    pa = synth.add_host_spread(s, 0.5).pod_affinity
    assert "task_xgroup_off" not in pa and "task_xgroup" not in pa and pa["n_groups"] == 16
    snap = aff_gen.random_affinity_session(3).flatten()
    assert "task_xgroup_off" not in snap.pod_affinity
    # above 32 labels the synthetic spread writes lists: label L >= 32 owns groups 2L, 2L + 1
    s, _ = synth.make("c1")
    pa = synth.add_host_spread(s, 1.0, labels=40).pod_affinity
    assert pa["n_groups"] == 80
    for f, c in group_sets(pa, s.T):
        assert f == c and len(f) == 2 and min(f) % 2 == 0 and max(f) == min(f) + 1
