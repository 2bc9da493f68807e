"""Sessions with more than 256 queues through the C ABI (-m gpu): the sessions of test_many_queues.py, bit-exact against the
oracle (decisions and dispatch steps, evictions in order, node / job / queue state, kb_bind_list), through the persistent
pipeline (R = 3, W = 2) and the per-visit kernels (R = 4); a C3-sized cluster in 1 000 queues against the emulation; and one
cluster with 300 queues through the C++ host mirror's cycle shells (tests/host/cycle_run) against kbo.cycle."""
from __future__ import annotations

import numpy as np
import pytest

from kube_batch_b200 import synth
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import util
from test_many_queues import ACTION_LISTS, FULL_LIST, deep_heap_session, many_queue_session, object_cluster, tier_variants

pytestmark = pytest.mark.gpu


def check_bind_list(eng, d, what):
    task, node = eng.bind_list()
    disp = np.nonzero(d["dispatched"] & (d["node"] >= 0))[0]
    order = disp[np.lexsort((d["step"][disp], d["dispatch_step"][disp]))]          # by dispatch step, then Allocate order
    np.testing.assert_array_equal(task, order.astype(np.uint32), err_msg=f"{what}: bind list tasks")
    np.testing.assert_array_equal(node, d["node"][order], err_msg=f"{what}: bind list nodes")


def check_cycle(eng, s, conf, acts, run, what):
    o, ev, order = kbo.cycle(s, conf, actions=acts, running=run)
    res, gev, gorder, bounds = eng.cycle(acts)
    np.testing.assert_array_equal(ev, gev, err_msg=f"{what}: evicted set")
    np.testing.assert_array_equal(order, gorder, err_msg=f"{what}: eviction order")
    util.assert_same_decisions(o.decisions, res.decisions, what)
    util.assert_same_state(o, eng.node_state(), eng.order_state(), what)
    check_bind_list(eng, o.decisions, what)
    assert int(bounds[-1][1]) == int(ev.sum())
    return res, int(ev.sum())


@pytest.mark.parametrize("Q", [256, 257, 300, 1000, 4096])
def test_many_queues_on_the_gpu(Q):
    from kube_batch_b200 import engine
    s, run = many_queue_session(Q, Q)
    eng = engine.Engine(0)
    evictions = 0
    for tname, conf in tier_variants():
        eng.load(s, conf).load_running(run)
        for acts in ACTION_LISTS:
            res, n = check_cycle(eng, s, conf, acts, run, f"Q={Q} {tname} {acts}")
            evictions += n
        o = kbo.allocate(s, conf)
        r = eng.allocate()
        util.assert_same_decisions(o.decisions, r.decisions, f"Q={Q} {tname} kb_allocate")
        assert int(r.stats.pipeline) == 1, "R = 3 / W = 2 sessions run the persistent pipeline"
    assert evictions > 0
    eng.close()


@pytest.mark.parametrize("Q", [300, 4096])
def test_many_queues_on_the_per_visit_kernels(Q):
    """R = 4: no cycle_kernel instance for that record geometry, so kb_allocate pumps the per-visit kernels."""
    from kube_batch_b200 import engine
    s = synth.random_session(Q, tasks=600, jobs=120, nodes=60, queues=Q, oversub=2.0, R=4)
    rng = np.random.default_rng(Q)
    s.queue_weight[:] = rng.integers(1, 101, size=Q)
    s.queue_ctime[:] = rng.integers(0, 3, size=Q)
    s.invalidate()
    eng = engine.Engine(0)
    for tname, conf in tier_variants():
        eng.load(s, conf)
        o = kbo.allocate(s, conf)
        r = eng.allocate()
        assert int(r.stats.pipeline) == 0
        util.assert_same_decisions(o.decisions, r.decisions, f"R=4 Q={Q} {tname}")
        util.assert_same_state(o, eng.node_state(), eng.order_state(), f"R=4 Q={Q} {tname}")
        check_bind_list(eng, o.decisions, f"R=4 Q={Q} {tname}")
    eng.close()


def test_queue_heap_deeper_than_12_levels_on_the_gpu():
    from kube_batch_b200 import engine
    s = deep_heap_session()
    eng = engine.Engine(0)
    for tname, conf in tier_variants():
        eng.load(s, conf)
        o = kbo.allocate(s, conf)
        r = eng.allocate()
        util.assert_same_decisions(o.decisions, r.decisions, f"deep heap {tname}")
        util.assert_same_state(o, eng.node_state(), eng.order_state(), f"deep heap {tname}")
    eng.close()


def test_c3_sized_cluster_in_1000_queues_on_the_gpu():
    """50 000 tasks, 5 000 PodGroups, 5 000 nodes, 1 000 queues: kb_allocate and the shipped action list against the emulation."""
    from kube_batch_b200 import engine
    s = synth.random_session(3, tasks=50_000, jobs=5_000, nodes=5_000, queues=1000, oversub=2.0)
    rng = np.random.default_rng(1000)
    s.queue_weight[:] = rng.integers(1, 101, size=1000)
    s.invalidate()
    run = synth.running_of(s, 0.4)
    conf = PluginConf.default()
    eng = engine.Engine(0)
    eng.load(s, conf).load_running(run)
    r = eng.allocate()
    g = util.emu_allocate(s, conf, mode=1)
    util.assert_same_decisions(g.decisions, r.decisions, "c3-sized allocate")
    assert int(r.stats.pipeline) == 1
    res, gev, gorder, bounds = eng.cycle(FULL_LIST)
    e, eev, eorder = util.emu_cycle(s, conf, FULL_LIST, run, mode=1)
    np.testing.assert_array_equal(eev, gev)
    np.testing.assert_array_equal(eorder, gorder)
    util.assert_same_decisions(e.decisions, res.decisions, "c3-sized cycle")
    util.assert_same_state(e, eng.node_state(), eng.order_state(), "c3-sized cycle")
    assert int(gev.sum()) > 0
    eng.close()


def test_cycle_shells_of_the_cpp_mirror_with_300_queues(tmp_path):
    import test_host_cpp_cycle as H
    H._build()
    b = object_cluster(7)
    cases = [(f"{tname}:{i}", acts, conf) for tname, conf in tier_variants() for i, acts in enumerate(ACTION_LISTS)]
    got = H.run_cases(tmp_path, b, cases)
    assert sorted(got) == sorted(label for label, _, _ in cases)
    evictions = [H.compare_with_oracle(b, got[label], acts, conf, f"300 queues {label} {acts}") for label, acts, conf in cases]
    assert sum(evictions) > 0, evictions
