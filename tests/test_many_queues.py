"""Sessions with more than 256 queues (up to KB_MAX_Q) against the oracle.

CPU: the host/device-shared algorithm run by tests/emu (launch modes 1 and 5) on seeded sessions this file builds: many queues
that own no job, equal creation times (the index / UID tie-break decides), weights from 1 to 100, tiers with and without
proportion and drf, and oversubscribed clusters with Running pods so that reclaim and preempt walk many queues.  The GPU twin
is test_gpu_many_queues.py."""
from __future__ import annotations

import numpy as np
import pytest

from kube_batch_b200 import abi, builder as B, synth
from kube_batch_b200.snapshot import PluginConf, PluginOption
from oracle import kbo
import util

FULL_LIST = ("reclaim", "allocate", "backfill", "preempt")            # config/kube-batch-conf.yaml:1
ACTION_LISTS = (("allocate",), ("allocate", "backfill"), FULL_LIST)


def tier_variants():
    t = True
    yield "default", PluginConf.default()
    yield "drf_first", PluginConf([[PluginOption("drf", enabled_job_order=t, enabled_preemptable=t),
                                    PluginOption("proportion", enabled_queue_order=t, enabled_reclaimable=t)],
                                   [PluginOption("gang", enabled_job_pipelined=t, enabled_preemptable=t, enabled_reclaimable=t),
                                    PluginOption("predicates", enabled_predicate=t), PluginOption("nodeorder", enabled_node_order=t)]])
    # no proportion, no drf: the queue heap orders by creation time and index only
    yield "no_fair_share", PluginConf([[PluginOption("priority", enabled_job_order=t, enabled_task_order=t, enabled_preemptable=t),
                                        PluginOption("gang", enabled_job_order=t, enabled_job_ready=t, enabled_job_pipelined=t,
                                                     enabled_preemptable=t, enabled_reclaimable=t),
                                        PluginOption("conformance", enabled_preemptable=t, enabled_reclaimable=t)],
                                       [PluginOption("predicates", enabled_predicate=t), PluginOption("nodeorder", enabled_node_order=t)]])


def many_queue_session(seed: int, Q: int, tasks: int = 600, jobs: int = 120, nodes: int = 60, oversub: float = 2.0, hot: int = 12):
    """synth.random_session with Q queues: weights 1..100, creation times from three values (many ties), half of the PodGroups in
    `hot` queues (several jobs per queue, so re-pushed jobs of one queue meet) and the rest spread over all Q (most queues own no
    job).  Returns (snapshot, Running tasks of the filler pods, 40 % of their PodGroups preemptable)."""
    s = synth.random_session(seed, tasks=tasks, jobs=jobs, nodes=nodes, queues=Q, oversub=oversub)
    rng = np.random.default_rng(90_000 + seed)
    s.queue_weight[:] = rng.integers(1, 101, size=Q)
    s.queue_ctime[:] = rng.integers(0, 3, size=Q)
    hot_q = rng.choice(Q, size=min(hot, Q), replace=False)
    jq = rng.integers(0, Q, size=jobs)
    half = rng.random(jobs) < 0.5
    jq[half] = rng.choice(hot_q, size=int(half.sum()))
    s.job_queue[:jobs] = jq
    s.invalidate()
    return s, synth.running_of(s, 0.4, seed=seed + 1)


def object_cluster(seed: int, nq: int = 300) -> B.SessionBuilder:
    """Running, terminating and Pending pods of PodGroups spread over `nq` queues, built from objects (queues named so that
    UID order differs from creation order in places)."""
    rng = np.random.default_rng(31_000 + seed)
    b = B.SessionBuilder()
    for q in range(nq):
        b.add_queue(B.Queue(f"q{q:05d}", int(rng.integers(1, 101)), creation=int(rng.integers(0, 3))))
    nn = int(rng.integers(20, 40))
    for n in range(nn):
        b.add_node(B.Node(f"n{n:04d}", {"cpu": 8, "memory": 32e9, "pods": int(rng.integers(6, 14))}))
    cap = {f"n{n:04d}": 8.0 for n in range(nn)}
    k = 0
    for g in range(int(rng.integers(60, 100))):
        b.add_pod_group(B.PodGroup("ns", f"g{g}", f"q{int(rng.integers(0, nq)):05d}", min_member=int(rng.integers(0, 4)),
                                   priority=int(rng.integers(0, 3)), creation=int(rng.integers(0, 4))))
        cpu = float(rng.choice([0.5, 1, 2, 3]))
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
            b.add_pod(B.Pod("ns", f"g{g}-p{i}", node, "Pending" if state == "Pending" else "Running", {"cpu": cpu, "memory": cpu * 1e9},
                            group=f"g{g}", priority=int(rng.integers(0, 3)), creation=k, deleting=(state == "Deleting")))
            k += 1
    return b


def deep_heap_session(Q: int = 5000, jobs: int = 9000):
    """One task per PodGroup, far more PodGroups than fit: the queue heap (one entry per job) holds 9000 entries, 14 levels."""
    s = synth.random_session(77, tasks=jobs, jobs=jobs, nodes=40, queues=Q, oversub=4.0)
    rng = np.random.default_rng(77)
    s.queue_weight[:] = rng.integers(1, 101, size=Q)
    s.queue_ctime[:] = 0
    s.invalidate()
    return s


def compare(what, o, ev, order, g, gev, gorder):
    np.testing.assert_array_equal(ev, gev, err_msg=f"{what}: evicted set")
    np.testing.assert_array_equal(order, gorder, err_msg=f"{what}: eviction order")
    util.assert_same_decisions(o.decisions, g.decisions, what)
    ns, os_ = util.emu_states(g)
    util.assert_same_state(o, ns, os_, what)


@pytest.mark.parametrize("Q", [256, 257, 300, 1000, 4096])
def test_many_queues_on_the_emulation(Q):
    s, run = many_queue_session(Q, Q)
    assert s.Q == Q and len(np.unique(s.job_queue)) < Q
    evictions = 0
    for tname, conf in tier_variants():
        for acts in ACTION_LISTS:
            o, ev, order = kbo.cycle(s, conf, actions=acts, running=run)
            for mode in (1, 5):
                g, gev, gorder = util.emu_cycle(s, conf, acts, run, mode=mode)
                compare(f"Q={Q} {tname} {acts} mode {mode}", o, ev, order, g, gev, gorder)
            evictions += int(ev.sum())
    assert evictions > 0, "some tier must make reclaim / preempt evict"


@pytest.mark.parametrize("seed", range(4))
def test_object_built_clusters_with_300_queues_on_the_emulation(seed):
    s = object_cluster(seed).flatten()
    assert s.Q == 300
    for tname, conf in tier_variants():
        for acts in ACTION_LISTS:
            o, ev, order = kbo.cycle(s, conf, actions=acts, running=s.meta["running"])
            g, gev, gorder = util.emu_cycle(s, conf, acts, s.meta["running"], mode=1 + 4 * (seed % 2))
            compare(f"seed {seed} {tname} {acts}", o, ev, order, g, gev, gorder)


def test_queue_heap_deeper_than_12_levels_on_the_emulation():
    s = deep_heap_session()
    assert s.J >= 8192                                     # qheap positions 8191.. are level 13 (the root is level 0)
    for tname, conf in tier_variants():
        o = kbo.allocate(s, conf)
        for mode in (1, 5):
            g, _, _ = util.emu_cycle(s, conf, ("allocate",), None, mode=mode)
            util.assert_same_decisions(o.decisions, g.decisions, f"deep heap {tname} mode {mode}")
            ns, os_ = util.emu_states(g)
            util.assert_same_state(o, ns, os_, f"deep heap {tname} mode {mode}")


def test_kb_max_q_queues_load_and_one_more_is_refused():
    assert abi.KB_MAX_Q == 65536
    s = synth.random_session(5, tasks=200, jobs=40, nodes=16, queues=abi.KB_MAX_Q)
    s.job_queue[:] = np.linspace(0, abi.KB_MAX_Q - 1, s.J).astype(s.job_queue.dtype)     # the first and the last queue own jobs
    s.invalidate()
    conf = PluginConf.default()
    o = kbo.allocate(s, conf)
    g = util.emu_allocate(s, conf, mode=1)
    util.assert_same_decisions(o.decisions, g.decisions, "Q = KB_MAX_Q")
    ns, os_ = util.emu_states(g)
    util.assert_same_state(o, ns, os_, "Q = KB_MAX_Q")

    s1 = synth.random_session(5, tasks=200, jobs=40, nodes=16, queues=abi.KB_MAX_Q + 1)
    with pytest.raises(RuntimeError, match=rf"rc={abi.KB_E_BADARG}\b.*KB_MAX_Q"):
        util.emu_allocate(s1, conf, mode=1)
