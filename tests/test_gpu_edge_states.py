"""`-m gpu`: the boundary-state sessions of tests/edge_gen.py through the C ABI, against the oracle, bit for bit.

The R = 3 / W = 2 sessions run on cycle_kernel, whose placement-depth chains the CPU emulation does not model: a list candidate
carries depths 0..7 evaluated up front, a patched one 0..3, and extend() evaluates 32 more depths into one shared buffer.  Runs of
more than 40 placements on one node need a second extension, 2..4 identical nodes under leastrequested make several deep candidates
alternate (their extensions evict each other), and pod caps / epsilon fits / Allocate -> Pipeline flips end the chains at chosen
depths.  The per-visit kernels (engine flags, R = 4 / W = 3), backfill, the full action list and the predicate / score matrices
run on the same sessions.  The counters the tests assert on are printed (-s)."""
import os

import numpy as np
import pytest

from kube_batch_b200 import abi, engine
from kube_batch_b200 import builder as B
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import edge_gen as E
import util
from test_edge_states import CYCLE, EDGE_CONFS, edge_confs
from test_emu_parity import CONFS
from test_evict_parity import compare
from test_gpu_parity import run_and_check, run_backfill_and_check

pytestmark = pytest.mark.gpu

PIPE_SESSIONS = [("base", 0, {}), ("base", 1, {}), ("base", 2, {}), ("multiqueue", 0, {"queues": 3}), ("pref", 0, {"pref": True}),
                 ("pref", 1, {"pref": True})]


def _session(variant, seed, kw):
    # the same seeds as tests/test_edge_states.py: a failure here and there points at the device, not at the shared logic
    return E.edge_session(100 * seed + len(variant), **kw)


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(device=0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def timed_eng():
    old = os.environ.get("KB_PIPE_TIMING")
    os.environ["KB_PIPE_TIMING"] = "1"          # read at engine creation: the pool-builder counters are kept in timing mode only
    try:
        e = engine.Engine(device=0)
    finally:
        if old is None:
            del os.environ["KB_PIPE_TIMING"]
        else:
            os.environ["KB_PIPE_TIMING"] = old
    yield e
    e.close()


def test_edge_sessions_on_the_persistent_pipeline(eng):
    extends = patched = 0
    covs = []
    for variant, seed, kw in PIPE_SESSIONS:
        s = _session(variant, seed, kw)
        for cname, conf in edge_confs():
            o, r = run_and_check(eng, s, conf, f"edge {variant}/seed{seed}/{cname}")
            assert r.stats.pipeline == 1, f"{variant}/seed{seed}/{cname}: the session did not run on cycle_kernel"
            extends += r.stats.pipe_extends
            patched += r.stats.pipe_patched
            covs.append(E.coverage(s, o))
    cov = E.merge(covs)
    print(f"\nedge sessions on cycle_kernel: pipe_extends {extends}, pipe_patched {patched}, coverage {cov}")
    E.assert_covered(cov, "pipeline sessions")
    assert extends > 0, "no candidate went past the depths evaluated up front"


def _one_node_runs(sizes, idle_tasks=None, releasing_tasks=0):
    """Jobs of one class, in a row, on ONE node (cpu 64, memory 256 Gi, 4 GPUs): each job is one run of its size (minMember = size).
    idle_tasks: room in Idle for that many tasks in all; releasing_tasks: that many more fit into Releasing (terminating pod)."""
    b = B.SessionBuilder()
    b.add_queue(B.Queue("q", 1))
    b.add_pod_group(B.PodGroup("ns", "old", "q", min_member=1))
    b.add_node(B.Node("n0", {"cpu": 64, "memory": 256 * E.GI, E.GPU: 4, "pods": 250}))
    req = {"cpu": 0.2, "memory": 256 * E.MI}
    if idle_tasks is not None:
        rel = {"cpu": 0.2 * releasing_tasks, "memory": 256 * E.MI * releasing_tasks}
        if releasing_tasks:
            b.add_pod(B.Pod("ns", "dying", "n0", "Running", rel, group="old", deleting=True))
        b.add_pod(B.Pod("ns", "busy", "n0", "Running", {"cpu": 64 - 0.2 * (idle_tasks + releasing_tasks), "memory": 4 * E.GI},
                        group="old"))
    for i, size in enumerate(sizes):
        b.add_pod_group(B.PodGroup("ns", f"j{i}", "q", min_member=size, creation=i))
        for k in range(size):
            b.add_pod(B.Pod("ns", f"j{i}-p{k:03d}", "", "Pending", dict(req), group=f"j{i}", creation=k))
    s = b.flatten(W=2)
    assert (s.R, s.W) == (3, 2)
    return s


@pytest.mark.parametrize("placements", [7, 8, 38, 39, 40, 41, 71, 72])
def test_extension_window_of_a_single_deep_candidate(eng, placements):
    """One job, one feasible node, `placements` tasks in one run: the candidate comes from the visit's list with depths 0..7
    evaluated up front; the replay extends it by depths 8..39 at its 8th placement and by 40..71 at its 40th.  The count pins the
    window of extend() (base = current depth + 1): a window that started one depth early would need its second extension at the
    39th placement, with the same decisions."""
    s = _one_node_runs([placements])
    o, r = run_and_check(eng, s, PluginConf.default(), f"one node x {placements}")
    assert int(o.result.tasks_allocated) == placements and r.stats.pipeline == 1
    want = int(placements >= 8) + int(placements >= 40) + int(placements >= 72)
    print(f"\n{placements} placements on one candidate: pipe_extends {r.stats.pipe_extends} (expected {want})")
    assert r.stats.pipe_extends == want


def test_relay_runs_on_one_node_end_at_every_shallow_depth(eng):
    """Jobs of one class in a row on one node: Idle ends the second job's run at depths 0..9 — around the end of the depths
    evaluated up front — with and without an Allocate -> Pipeline flip onto Releasing before the node stops fitting."""
    for first in (1, 2, 3, 5):
        for end in range(0, 10):
            for rel in (0, 3):
                s = _one_node_runs([first, 40, 40], idle_tasks=first + end, releasing_tasks=rel)
                o, r = run_and_check(eng, s, PluginConf.default(), f"relay first {first} end {end} releasing {rel}")
                assert int(o.result.tasks_allocated) == first + end and int(o.result.tasks_pipelined) == rel


def test_edge_sessions_pool_builder_paths(timed_eng):
    used = missed = cancelled = 0
    for variant, seed, kw in PIPE_SESSIONS:
        s = _session(variant, seed, kw)
        for cname in ("default", "c2", "weights"):
            o, r = run_and_check(timed_eng, s, CONFS[cname], f"edge timed {variant}/seed{seed}/{cname}")
            assert r.stats.pipeline == 1
            used += r.stats.pipe_builds_used
            missed += r.stats.pipe_builds_missed
            cancelled += r.stats.pipe_builds_cancelled
    print(f"\nedge sessions, pool builder: used {used}, missed {missed}, cancelled {cancelled}")
    assert used > 0 and missed > 0 and cancelled > 0, (used, missed, cancelled)


@pytest.mark.parametrize("flag", [abi.KB_ENGINE_NO_PIPE, abi.KB_ENGINE_CHAIN2, abi.KB_ENGINE_CHAIN4, abi.KB_ENGINE_FORCE_OVERLAP],
                         ids=["no_pipe", "chain2", "chain4", "force_overlap"])
def test_edge_sessions_on_the_per_visit_kernels(flag):
    e = engine.Engine(device=0, flags=flag | (abi.KB_ENGINE_NO_PIPE if flag != abi.KB_ENGINE_NO_PIPE else 0))
    try:
        for variant, seed, kw in PIPE_SESSIONS[:4]:
            s = _session(variant, seed, kw)
            for cname in EDGE_CONFS:
                o, r = run_and_check(e, s, CONFS[cname], f"edge flag{flag} {variant}/seed{seed}/{cname}")
                assert r.stats.pipeline == 0
    finally:
        e.close()


def test_edge_sessions_wide_records(eng):
    """R = 4 / W = 3: a fourth resource and a third mask word, outside cycle_kernel's geometry."""
    covs = []
    for seed in range(3):
        s = _session("wide", seed, {"wide": True})
        assert (s.R, s.W) == (4, 3)
        for cname, conf in edge_confs():
            o, r = run_and_check(eng, s, conf, f"edge wide/seed{seed}/{cname}")
            assert r.stats.pipeline == 0
            covs.append(E.coverage(s, o))
    E.assert_covered(E.merge(covs), "wide sessions")


@pytest.mark.parametrize("seed", range(3))
def test_edge_sessions_backfill(eng, seed):
    s = E.edge_session(300 + seed, queues=1 + seed % 2, best_effort=True)
    for cname in ("default", "c2", "weights", "allocate_test"):
        for actions in (2, 3):
            run_backfill_and_check(eng, s, CONFS[cname], f"edge backfill seed{seed}/{cname}/actions{actions}", actions)


@pytest.mark.parametrize("seed", range(4))
def test_edge_sessions_full_action_list(eng, seed):
    s = E.edge_session(500 + seed, queues=1 + seed % 3, best_effort=seed % 2 == 1, long_runs=seed < 2)
    run = s.meta["running"]
    for cname, conf in (("default", PluginConf.default()), ("c2", CONFS["c2"]), ("weights", CONFS["weights"])):
        o, ev, order = kbo.cycle(s, conf, actions=CYCLE, running=run)
        eng.load(s, conf).load_running(run)
        res, gev, gorder, _ = eng.cycle(CYCLE)
        what = f"edge cycle seed{seed}/{cname}"
        compare(what, o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
        util.assert_same_decisions(o.decisions, res.decisions, what)


@pytest.mark.parametrize("seed", range(2))
def test_edge_predicate_score_and_best_nodes(eng, seed):
    """kb_predicate_score / kb_best_nodes on the loaded boundary states: fit and score of every (task, node) against the oracle."""
    s = _session("base", seed, {})
    for cname in ("default", "weights", "negweight"):
        conf = CONFS[cname] if cname != "weights" else E.mostrequested_conf()
        eng.load(s, conf)
        fit, score = eng.predicate_score(0, s.T)
        rows = list(range(0, s.T, 3)) + [s.T - 1]
        for t in rows:
            of, osc = kbo.predicate_score(s, conf, t)
            np.testing.assert_array_equal(of, fit[t], err_msg=f"{cname} fit row {t}")
            np.testing.assert_array_equal(osc, score[t], err_msg=f"{cname} score row {t}")
        best = engine.key_node(eng.best_nodes(0, s.T))
        masked = np.where(fit > 0, score, -np.inf)
        exp = np.where(fit.any(axis=1), masked.argmax(axis=1), -1)
        np.testing.assert_array_equal(exp, best, err_msg=cname)
        assert (fit.any(axis=1)).sum() > s.T // 2 and not fit.all()
