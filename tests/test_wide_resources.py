"""Sessions with 9 to 32 resource dimensions (KB_MAX_R) against the oracle.

The engine runs such sessions on the kernels' wide instances (class records of KB_MAX_R dimensions).  CPU: the same algorithm
run by the emulation built with wide class records (tests/emu_wide: tests/emu/kb_emu.cpp with KB_CLASS_R = KB_MAX_R) in every
launch mode, on seeded synthetic sessions, object clusters with Running pods, affinity sessions and hand-computed cases whose
deciding resource sits at a high dimension index.  The GPU twin is test_gpu_wide_resources.py."""
from __future__ import annotations

import contextlib
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from kube_batch_b200 import abi, builder as B, synth
from kube_batch_b200.snapshot import PluginConf, PluginOption
from oracle import kbo
import aff_gen
import util
from test_evict_parity import compare, random_cluster, tier_variants

_HERE = os.path.dirname(os.path.abspath(__file__))
FULL_LIST = ("reclaim", "allocate", "backfill", "preempt")            # config/kube-batch-conf.yaml:1
ACTION_LISTS = (("allocate",), ("allocate", "backfill"), FULL_LIST)
EMU_MODES = (0, 1, 2, 4, 5)                                           # overlap, plain, chained x2 / x4, persistent pipeline
SCALARS = [f"example.com/s{i:02d}" for i in range(30)]               # dims 2..31 in name order: s{k-2} is dimension k
_wide = None


def wide_lib():
    global _wide
    if _wide is None:
        d = os.path.join(_HERE, "emu_wide")
        with open(os.path.join(d, ".build.lock"), "w") as lk:
            import fcntl
            fcntl.flock(lk, fcntl.LOCK_EX)
            subprocess.check_call(["make", "-C", d, "-s"])
        _wide = C.CDLL(os.path.join(d, "libkbemu_wide.so"))
        _wide.kbemu_last_error.restype = C.c_char_p
    return _wide


@contextlib.contextmanager
def wide_emulation():
    """util's emulation helpers, run by the emulation with wide class records"""
    saved = util._emu
    util._emu = wide_lib()
    try:
        yield
    finally:
        util._emu = saved


def widen(b: B.SessionBuilder, R: int, seed: int) -> B.SessionBuilder:
    """Adds R - 2 - (scalars already named) scalar resources: on about half of the nodes (a third of those at value 0, the
    rest with 1..8 units), requested by about a fifth of the Pending pods (one or two of them) and by about a third of the Running
    pods (one unit of one of them, the node's Allocatable raised to what its Running pods hold), so that reclaim / preempt pick
    victims whose requests reach past dimension 8."""
    rng = np.random.default_rng(4400 + seed)
    have = {k for n in b.nodes for k in n.allocatable if k not in ("cpu", "memory", "pods")}
    have |= {k for p in b.pods for k in p.requests if k not in ("cpu", "memory", "pods")}
    extra = [s for s in SCALARS if s not in have][: R - 2 - len(have)]
    for n in b.nodes:
        for s in extra:
            if rng.random() < 0.5:
                n.allocatable[s] = 0.0 if rng.random() < 0.33 else float(rng.integers(1, 9))
    for s in extra:                                                   # every name is listed by some node
        if not any(s in n.allocatable for n in b.nodes):
            b.nodes[0].allocatable[s] = 0.0
    held = {}                                                         # (node, scalar) -> units Running pods hold
    for p in b.pods:
        if not extra or rng.random() >= (0.3 if p.node_name else 0.2):
            continue
        p.requests = dict(p.requests)
        for s in rng.choice(extra, size=min(len(extra), 1 if p.node_name else int(rng.integers(1, 3))), replace=False):
            p.requests[str(s)] = 1.0
            if p.node_name:
                held[(p.node_name, str(s))] = held.get((p.node_name, str(s)), 0) + 1
    by_name = {n.name: n for n in b.nodes}
    for (nn, s), k in held.items():                                   # the node lists what its Running pods hold: Idle stays >= 0
        n = by_name[nn]
        n.allocatable[s] = max(float(n.allocatable.get(s, 0.0)), float(k))
    return b


def check_cycle(s, tiers, acts, running, what, modes=EMU_MODES):
    o, ev, order = kbo.cycle(s, tiers, actions=acts, running=running)
    with wide_emulation():
        for mode in modes:
            g, gev, gorder = util.emu_cycle(s, tiers, acts, running, mode=mode)
            compare(f"{what} mode {mode}", o, ev, order, g, gev, gorder, util.emu_states(g))
            util.assert_same_decisions(o.decisions, g.decisions, f"{what} mode {mode}")
    return o, ev, order


# ------------------------------------------------------------------------------------------------ random sessions
@pytest.mark.parametrize("R", [9, 12, 17, 32])
@pytest.mark.parametrize("seed", range(2))
def test_synthetic_sessions_on_the_emulation(R, seed):
    s = synth.random_session(seed, tasks=300, jobs=40, nodes=40, queues=2, oversub=3.0, R=R)
    run = synth.running_of(s, 0.8, seed=seed + 1)
    evictions = 0
    for tname, tiers in tier_variants():
        for acts in ACTION_LISTS:
            o, ev, _ = check_cycle(s, tiers, acts, run, f"R {R} seed {seed} {tname} {acts}")
            evictions += int(ev.sum())
    assert s.R == R and evictions > 0


CLUSTER_SEEDS = range(4)


@pytest.mark.parametrize("R", [9, 12, 17, 32])
@pytest.mark.parametrize("seed", CLUSTER_SEEDS)
def test_object_clusters_with_running_pods_on_the_emulation(R, seed):
    s = widen_cluster(seed, R)
    assert s.R == R
    for tname, tiers in tier_variants():
        for acts in ACTION_LISTS:
            check_cycle(s, tiers, acts, s.meta["running"], f"R {R} cluster {seed} {tname} {acts}", modes=(1, 5))


@pytest.mark.parametrize("R", [17, 32])
def test_the_object_clusters_evict_victims_past_dimension_8(R):
    """what the clusters above (and their GPU twins) exercise: victims whose requests reach past the narrow class record"""
    high = 0
    for seed in CLUSTER_SEEDS:
        s = widen_cluster(seed, R)
        for tname, tiers in tier_variants():
            for acts in ACTION_LISTS:
                high += evicted_high(s, kbo.cycle(s, tiers, actions=acts, running=s.meta["running"])[1])
    assert high > 0


def evicted_high(s, ev) -> int:
    """victims that hold a resource in dimension 8 or above (past the narrow class record)"""
    rq = np.asarray(s.meta["running"]["resreq"])
    return int((np.asarray(ev, dtype=bool) & (rq[8:].sum(axis=0) > 0)).sum()) if rq.shape[0] > 8 else 0


def widen_cluster(seed: int, R: int):
    """test_evict_parity's random cluster (Running, terminating and Pending pods) with R dimensions"""
    b = random_cluster_builder(seed)
    return widen(b, R, seed).flatten()


def random_cluster_builder(seed: int) -> B.SessionBuilder:
    # random_cluster builds and flattens; rebuild the same objects through a builder that keeps them
    orig = B.SessionBuilder.flatten
    box = {}

    def keep(self):
        box["b"] = self
        return orig(self)
    B.SessionBuilder.flatten = keep
    try:
        random_cluster(seed)
    finally:
        B.SessionBuilder.flatten = orig
    return box["b"]


def affinity_session(seed: int):
    """preferred node affinity (node_pref, even seeds) and inter-pod terms (aff_gen) with 12 dimensions"""
    s = widen(aff_gen.random_affinity_session(seed, n_nodes=16, n_groups=8, node_pref=(seed % 2 == 0)), 12, seed).flatten()
    assert s.R == 12
    return s


# reclaim / preempt refused in a session whose pending classes read counter groups, or withheld after a group member's eviction
REFUSED_EVICT = ("outside this build", "the outcome of this cycle is withheld")


@pytest.mark.parametrize("seed", range(6))
def test_affinity_sessions_at_12_dimensions_on_the_emulation(seed):
    s = affinity_session(seed)
    for tname, tiers in tier_variants():
        for acts in ACTION_LISTS:
            try:
                check_cycle(s, tiers, acts, s.meta.get("running"), f"affinity {seed} {tname} {acts}")
            except RuntimeError as e:
                assert acts == FULL_LIST and any(m in str(e) for m in REFUSED_EVICT), e


# ------------------------------------------------------------------------------------------------ hand-computed cases
def scalar_node(name, cpu=8, mem=32e9, **scalars):
    a = {"cpu": cpu, "memory": mem, "pods": 110}
    a.update(scalars)
    return B.Node(name, a)


def all_scalars_builder(nodes, queues=("q0",)):
    """Every one of SCALARS is named by some node (the extra node `zz-all`, listing them all at 0), so that s{k-2} is dim k"""
    b = B.SessionBuilder()
    for q in queues:
        b.add_queue(B.Queue(q, 1))
    for n in nodes:
        b.add_node(n)
    b.add_node(scalar_node("zz-all", cpu=0, mem=0, **{s: 0.0 for s in SCALARS}))
    return b


def place(s, tiers, acts=("allocate",), running=None):
    o, ev, order = check_cycle(s, tiers, acts, running if running is not None else s.meta.get("running"), "hand case")
    return o, ev


PRED_ONLY = PluginConf([[PluginOption("predicates", enabled_predicate=True)]])


def case_a_request_in_dimension_20_on_a_node_without_a_scalar_map_and_with_a_zero(run):
    """resource_info.go:268-300: a scalar request <= 10 milli is skipped; a larger one fits neither a node whose ScalarResources
    is nil (`rr == nil -> false`) nor one where the scalar is present at 0."""
    s20 = SCALARS[18]
    for req, fits in ((0.005, True), (0.010, True), (1.0, False)):
        b = all_scalars_builder([scalar_node("a-nil"), scalar_node("b-zero", **{s20: 0.0})])
        b.add_pod_group(B.PodGroup("ns", "g", "q0", min_member=1))
        b.add_pod(B.Pod("ns", "p", requests={"cpu": 1, "memory": 1e9, s20: req}, group="g"))
        s = b.flatten()
        assert s.R == 32
        o, _ = run(s, PRED_ONLY)
        assert (o.decisions["kind"][0] == abi.KB_KIND_ALLOCATED) == fits, (req, o.decisions[0])
        if fits:
            assert o.decisions["node"][0] == 0                           # "a-nil": first in name order, equal scores


def case_a_request_within_10_milli_of_idle_in_dimension_31(run):
    s31 = SCALARS[29]
    for req, fits in ((2.009, True), (2.011, False)):
        b = all_scalars_builder([scalar_node("a", **{s31: 2.0})])
        b.add_pod_group(B.PodGroup("ns", "g", "q0", min_member=1))
        b.add_pod(B.Pod("ns", "p", requests={"cpu": 1, "memory": 1e9, s31: req}, group="g"))
        s = b.flatten()
        o, _ = run(s, PRED_ONLY)
        assert (o.decisions["kind"][0] == abi.KB_KIND_ALLOCATED) == fits, req


def case_a_drf_dominant_share_decided_by_dimension_25(run):
    """Job A holds 10 % of the cpu and 80 % of s23 (dim 25), job B 50 % of the cpu: drf orders B first, and only one of their
    pending pods fits.  Without dimension 25 A's share would be 0.1 and A would go first."""
    s25 = SCALARS[23]
    b = all_scalars_builder([scalar_node("a", cpu=10, mem=100e9, **{s25: 10.0})])
    for g in ("ga", "gb"):
        b.add_pod_group(B.PodGroup("ns", g, "q0", min_member=1))
    b.add_pod(B.Pod("ns", "ra", "a", "Running", {"cpu": 1, "memory": 1e9, s25: 8.0}, group="ga"))
    b.add_pod(B.Pod("ns", "rb", "a", "Running", {"cpu": 5, "memory": 1e9}, group="gb"))
    b.add_pod(B.Pod("ns", "pa", requests={"cpu": 4, "memory": 1e9}, group="ga"))
    b.add_pod(B.Pod("ns", "pb", requests={"cpu": 4, "memory": 1e9}, group="gb"))
    s = b.flatten()
    tiers = PluginConf([[PluginOption("drf", enabled_job_order=True)], [PluginOption("predicates", enabled_predicate=True)]])
    o, _ = run(s, tiers)
    kinds = o.decisions["kind"]                                      # jobs in JobID order: ns/ga, ns/gb; tasks pa, pb
    assert kinds[1] == abi.KB_KIND_ALLOCATED and kinds[0] == abi.KB_KIND_NONE, o.decisions
    assert o.job_share[0] == pytest.approx(0.8)                      # job A's dominant share: dimension 25


def case_a_queue_whose_only_request_is_in_dimension_30(run):
    """proportion (proportion.go:100-154): q1's pods ask for s28 (dim 30) only, 3 units in all; the round robin gives each of the
    two queues (equal weights) half of the 4 units.  q1's Running pod holds 2 of them, but Overused (deserved <= allocated) also
    reads cpu and memory, which q1 holds none of: q1 is not overused and both pending pods are placed."""
    s30 = SCALARS[28]
    b = all_scalars_builder([scalar_node("a", cpu=8, mem=32e9, **{s30: 4.0})], queues=("q0", "q1"))
    b.add_pod_group(B.PodGroup("ns", "g0", "q0", min_member=1))
    b.add_pod_group(B.PodGroup("ns", "g1", "q1", min_member=1))
    b.add_pod(B.Pod("ns", "r1", "a", "Running", {s30: 2.0}, group="g1"))
    b.add_pod(B.Pod("ns", "p1", requests={s30: 1.0}, group="g1"))
    b.add_pod(B.Pod("ns", "p0", requests={"cpu": 1, "memory": 1e9}, group="g0"))
    s = b.flatten()
    o, _ = run(s, PluginConf.default())
    d30 = o.queue_deserved[30]
    assert d30[0] == 2000.0 and d30[1] == 2000.0                     # milli
    kinds = o.decisions["kind"]                                      # jobs in JobID order: ns/g0 (p0), ns/g1 (p1)
    assert (kinds == abi.KB_KIND_ALLOCATED).all(), o.decisions
    assert o.queue_allocated[30][1] == 3000.0


def case_victims_that_cover_the_request_only_through_dimension_17(run, action):
    """The pending pod fits everywhere but in s15 (dim 17), which only the victim's eviction frees."""
    s17 = SCALARS[15]
    b = all_scalars_builder([scalar_node("a", cpu=16, mem=64e9, **{s17: 4.0})], queues=("q0", "q1"))
    q_victim, q_pre = ("q0", "q1") if action == "reclaim" else ("q0", "q0")
    b.add_pod_group(B.PodGroup("ns", "gv", q_victim, min_member=1, priority=0))
    b.add_pod_group(B.PodGroup("ns", "gp", q_pre, min_member=1, priority=2))
    b.add_pod(B.Pod("ns", "v", "a", "Running", {"cpu": 1, "memory": 1e9, s17: 4.0}, group="gv", priority=0))
    b.add_pod(B.Pod("ns", "p", requests={"cpu": 1, "memory": 1e9, s17: 4.0}, group="gp", priority=2))
    s = b.flatten()
    tiers = PluginConf([[PluginOption("priority", enabled_job_order=True, enabled_preemptable=True),
                         PluginOption("conformance", enabled_preemptable=True, enabled_reclaimable=True)],
                        [PluginOption("predicates", enabled_predicate=True)]])
    o, ev = run(s, tiers, acts=(action,), running=s.meta["running"])
    assert int(ev.sum()) == 1
    assert o.decisions["kind"][0] == abi.KB_KIND_PIPELINED


HAND_CASES = [case_a_request_in_dimension_20_on_a_node_without_a_scalar_map_and_with_a_zero,
              case_a_request_within_10_milli_of_idle_in_dimension_31, case_a_drf_dominant_share_decided_by_dimension_25,
              case_a_queue_whose_only_request_is_in_dimension_30,
              lambda run: case_victims_that_cover_the_request_only_through_dimension_17(run, "reclaim"),
              lambda run: case_victims_that_cover_the_request_only_through_dimension_17(run, "preempt")]
HAND_IDS = ["dim20_fit", "dim31_epsilon", "dim25_drf", "dim30_proportion", "dim17_reclaim", "dim17_preempt"]


@pytest.mark.parametrize("case", HAND_CASES, ids=HAND_IDS)
def test_hand_computed_cases_on_the_emulation(case):
    """the oracle and the emulation agree, and the oracle gives the hand-computed outcome"""
    case(place)


# ------------------------------------------------------------------------------------------------ objects to tables
def mig_cluster() -> B.SessionBuilder:
    """Zero-valued hugepages-*, attachable-volumes-*, MIG profiles next to nvidia.com/gpu, RDMA and SR-IOV devices (15 dims);
    pending pods request subsets of them, Running pods hold MIG slices and devices"""
    names = ["hugepages-1Gi", "hugepages-2Mi", "attachable-volumes-aws-ebs", "nvidia.com/gpu"] + \
            [f"nvidia.com/mig-{p}" for p in ("1g.10gb", "1g.20gb", "2g.20gb", "3g.40gb", "4g.40gb", "7g.80gb")] + \
            ["rdma/hca", "openshift.io/sriov-a", "openshift.io/sriov-b"]
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q0", 1))
    for i in range(4):
        a = {"cpu": 64, "memory": 512e9, "pods": 110, "hugepages-1Gi": 0.0, "hugepages-2Mi": 0.0, "attachable-volumes-aws-ebs": 25}
        if i % 2 == 0:
            a.update({"nvidia.com/mig-1g.10gb": 7, "nvidia.com/mig-2g.20gb": 3, "nvidia.com/mig-3g.40gb": 2, "nvidia.com/mig-7g.80gb": 1,
                      "nvidia.com/mig-1g.20gb": 0.0, "nvidia.com/mig-4g.40gb": 0.0, "nvidia.com/gpu": 0.0})
        else:
            a.update({"nvidia.com/gpu": 8, "rdma/hca": 1, "openshift.io/sriov-a": 4, "openshift.io/sriov-b": 4})
        b.add_node(B.Node(f"n{i}", a))
    b.add_pod_group(B.PodGroup("ns", "g", "q0", min_member=1))
    reqs = [{"nvidia.com/mig-1g.10gb": 1}, {"nvidia.com/gpu": 2, "rdma/hca": 1}, {"nvidia.com/mig-3g.40gb": 1, "hugepages-2Mi": 0.5},
            {"openshift.io/sriov-b": 1}, {"nvidia.com/mig-7g.80gb": 1}]
    for k, r in enumerate(reqs):
        b.add_pod(B.Pod("ns", f"p{k}", requests=dict({"cpu": 1, "memory": 1e9}, **r), group="g"))
    b.add_pod_group(B.PodGroup("ns", "run", "q0", min_member=1))
    for k, (node, r) in enumerate([("n0", {"nvidia.com/mig-7g.80gb": 1}), ("n0", {"nvidia.com/mig-1g.10gb": 3}),
                                   ("n1", {"nvidia.com/gpu": 6, "rdma/hca": 1}), ("n2", {"nvidia.com/mig-3g.40gb": 2})]):
        b.add_pod(B.Pod("ns", f"r{k}", node, "Running", dict({"cpu": 2, "memory": 4e9}, **r), group="run"))
    return b, names, reqs


def test_flatten_zero_valued_hugepages_volumes_and_mig_profiles(tmp_path):
    b, names, reqs = mig_cluster()
    s = b.flatten()
    dims = sorted(names)
    assert s.R == 2 + len(dims) == 15
    for i in range(4):                                                # the zero-valued entries are present (api.NewResource)
        for k, nm in enumerate(dims):
            listed = nm in b.nodes[i].allocatable
            assert bool((int(s.node_alloc_present[i]) >> (k + 2)) & 1) == listed, (i, nm)
    for t, r in enumerate(reqs):
        for k, nm in enumerate(dims):
            assert bool((int(s.task_res_present[t]) >> (k + 2)) & 1) == (nm in r), (t, nm)
    for tname, tiers in tier_variants():
        for acts in ACTION_LISTS:
            check_cycle(s, tiers, acts, s.meta["running"], f"mig cluster {tname} {acts}", modes=(1,))


def test_the_cpp_mirror_flattens_the_mig_cluster_like_builder(tmp_path):
    """kbhost.hpp's Flatten / FlattenRunning (tests/host cycle_run --running, affinity_run --flat; no GPU) on the same objects:
    the same dimensions in the same order, the Running table's requests and presence masks dimension for dimension"""
    import test_host_cpp_affinity as HA
    import test_host_cpp_cycle as HC
    HC._build()
    HA._build()
    b, names, _ = mig_cluster()
    rt = HC.check_running_table(tmp_path, b)
    assert np.asarray(rt["resreq"]).shape[0] == 2 + len(names)
    HA.check_flat(tmp_path, b)


# ------------------------------------------------------------------------------------------------ refusals
def test_more_than_32_dimensions_are_refused():
    s = synth.random_session(1, tasks=40, jobs=6, nodes=8, R=32)
    cs, keep = s.to_c()
    cs.R = abi.KB_MAX_R + 1
    s.to_c = lambda: (cs, keep)
    with wide_emulation(), pytest.raises(RuntimeError, match=r"rc=-1: R=33 / W=2 out of range \(2 <= R <= KB_MAX_R = 32"):
        util.emu_allocate(s, PluginConf.default())


def _sharded_rank(rank, world, port, R, q):
    import util as U
    import test_wide_resources as W
    U._emu = W.wide_lib()
    s = synth.random_session(2, tasks=60, jobs=8, nodes=300, R=R)
    try:
        out = U.emu_sharded_rank(rank, world, port, s, PluginConf.default())
        ref = kbo.allocate(s, PluginConf.default())
        U.assert_same_decisions(ref.decisions, out.decisions, f"R={R} rank {rank}")
        q.put((rank, "ok"))
    except Exception as e:                                                    # noqa: BLE001 — the message travels to the parent
        q.put((rank, str(e)))


@pytest.mark.parametrize("R", [8, 9])
def test_a_sharded_gloo_world_of_two(R):
    """A sharded node axis takes R <= 8 (the exchange's records); R = 9 is refused on every rank, naming the limit"""
    import multiprocessing as mp
    import socket
    sk = socket.socket()
    sk.bind(("127.0.0.1", 0))
    port = sk.getsockname()[1]
    sk.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_rank, args=(r, 2, port, R, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    for rank in range(2):
        if R <= 8:
            assert res[rank] == "ok", res
        else:
            assert "R=9 resource dimensions with a sharded node axis (KB_ENGINE_SHARD)" in res[rank], res
            assert "at most 8 dimensions" in res[rank], res


def test_the_narrow_emulation_refuses_wide_sessions():
    """host code that reads the class table as 8-dimension records (tests/emu) is told so instead of misreading a wide table"""
    s = synth.random_session(3, tasks=40, jobs=6, nodes=8, R=9)
    with pytest.raises(RuntimeError, match="class records of 8 resource dimensions"):
        util.emu_allocate(s, PluginConf.default())
