"""`-m gpu`: sessions with more than 64 inter-pod affinity counter groups through the C ABI (visit_kernel<BF, AFF = 1> with the
forbidden-group lists staged in shared memory, aff_prepass_kernel, cycle_kernel for host-level groups as atoms), against the
object-level oracle; at BASELINE size against the emulation."""
import json
import os

import numpy as np
import pytest

from kube_batch_b200 import abi, engine, synth
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import aff_gen_many
import util
import test_pod_affinity as tpa
from test_many_aff_groups import atoms_fit, forty_apps, many_owners, relabel, _with, FORBID

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(device=0)
    yield e
    e.close()


def run_and_check(eng, snap, conf, what, actions=1, pipeline=0):
    o = kbo.allocate(snap, conf, actions=actions)
    eng.load(snap, conf)
    r = eng.allocate()
    assert r.stats.pipeline == pipeline, what
    if actions & 2:
        r = eng.backfill()
    util.assert_same_decisions(o.decisions, r.decisions, what)
    util.assert_same_state(o, eng.node_state(), eng.order_state(), what)
    return o, r


@pytest.mark.parametrize("replica_node,expect", [("n0", 1), ("n1", 0)])
def test_only_a_group_above_63_decides_on_the_gpu(eng, replica_node, expect):
    snap = forty_apps(replica_node)
    t39 = snap.meta["tasks"].index("ns/a39")
    for ci, conf in enumerate(tpa.AFF_CONFS):
        o, r = run_and_check(eng, snap, conf, f"replica on {replica_node} conf {ci}", actions=3)
        if ci == 0:
            assert int(r.decisions["node"][t39]) == expect


@pytest.mark.parametrize("case", range(2))
def test_relabelled_sessions_on_the_gpu(eng, case):
    snap = forty_apps("n0") if case == 0 else aff_gen_many.random_affinity_session(51, n_nodes=11, n_groups=120, n_apps=48).flatten()
    NG = int(snap.pod_affinity["n_groups"])
    r = relabel(snap, np.arange(NG)[::-1].copy())
    for ci, conf in enumerate(tpa.AFF_CONFS):
        run_and_check(eng, snap, conf, f"case {case} conf {ci}", actions=3)
        run_and_check(eng, r, conf, f"case {case} conf {ci} relabelled", actions=3)


@pytest.mark.parametrize("seed", range(12))
def test_random_sessions_with_many_groups_on_the_gpu(eng, seed):
    snap = aff_gen_many.random_affinity_session(seed, n_nodes=6 + seed % 13, n_groups=100 + 10 * (seed % 5), n_apps=40 + 4 * (seed % 6),
                                           besteffort=seed % 4 == 3).flatten()
    assert 65 <= snap.pod_affinity["n_groups"] <= 300
    for ci, conf in enumerate(tpa.AFF_CONFS):
        run_and_check(eng, snap, conf, f"seed {seed} conf {ci}", actions=1)
        run_and_check(eng, snap, conf, f"seed {seed} conf {ci} +backfill", actions=3)


def test_a_class_forbidden_by_more_groups_than_the_scan_stages(eng):
    """the scan reads the forbidden-group list beyond its shared-memory bound (AFF_XF_SMEM = 128 entries) from L2"""
    snap = many_owners()
    pa = snap.pod_affinity
    assert pa["n_groups"] == 200 and int(pa["task_xgroup_off"][1]) == 136
    for ci, conf in enumerate(tpa.AFF_CONFS[:3]):
        o, r = run_and_check(eng, snap, conf, f"conf {ci}", actions=3)
        assert (r.decisions["kind"] == abi.KB_KIND_ALLOCATED).all() and (r.decisions["node"] >= 200).all()


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("fit", [True, False])
def test_host_spread_with_many_groups_on_the_gpu(eng, seed, fit):
    n_apps, n_pg = (40, 80) if fit else (120, 150)
    snap = aff_gen_many.host_spread_session(900 + seed, n_nodes=6 + seed % 11, n_groups=n_pg, pipe_geometry=True, ports=seed % 3 == 0,
                                       n_apps=n_apps).flatten(W=2)
    if fit and snap.pod_affinity["n_groups"] <= 64:
        pytest.skip("fewer than 65 groups drawn")
    assert atoms_fit(snap) == fit
    for ci, conf in enumerate((PluginConf.default(), PluginConf.from_names([["gang"], ["predicates"]]))):
        for actions in (1, 3):
            run_and_check(eng, snap, conf, f"seed {seed} conf {ci} actions {actions}", actions=actions, pipeline=1 if fit else 0)


@pytest.mark.parametrize("seed", range(6))
def test_shipped_action_list_with_many_groups_on_the_gpu(eng, seed):
    from test_evict_parity import tier_variants
    acts = ("reclaim", "allocate", "backfill", "preempt")
    for members in (False, True):
        s = aff_gen_many.evict_spread_cluster(seed, members_running=members, n_apps=300, n_pod_groups=90, W=2)
        assert s.pod_affinity["n_groups"] > 64
        member = (s.meta["running"]["flags"] & abi.KB_RUNNING_AFF_MEMBER) != 0
        for tname, tiers in tier_variants():
            o, ev, order = kbo.cycle(s, tiers, actions=acts, running=s.meta["running"])
            eng.load(s, tiers)
            eng.load_running(s.meta["running"])
            try:
                r, gev, gorder, _ = eng.cycle(acts)
            except engine.KbError as ex:
                assert members and ex.code == abi.KB_E_UNSUPPORTED_FEATURE and "withheld" in str(ex)
                continue
            np.testing.assert_array_equal(ev, gev, err_msg=f"seed {seed} {tname}: evicted set")
            np.testing.assert_array_equal(order, gorder, err_msg=f"seed {seed} {tname}: eviction order")
            util.assert_same_decisions(o.decisions, r.decisions, f"seed {seed} members {members} {tname}")
            util.assert_same_state(o, eng.node_state(), eng.order_state(), f"seed {seed} members {members} {tname}")
            assert not (gev & member).any()


def test_refusals_through_the_c_abi(eng):
    snap = forty_apps("n0")
    pa = snap.pod_affinity
    G = abi.KB_MAX_AFF_GROUPS + 1
    cases = [(abi.KB_E_UNSUPPORTED_FEATURE, dict(n_groups=G, group_keyset=np.zeros(G, np.uint32), group_total0=np.zeros(G, np.int32),
                                                  group_count0=np.zeros(G * snap.N, np.int32))),
             (abi.KB_E_BADARG, dict(task_xgroup=None))]
    for bad in ((5 << 2) | FORBID, (80 << 2) | FORBID):
        x = np.array(pa["task_xgroup"]); x[0] = bad
        cases.append((abi.KB_E_BADARG, dict(task_xgroup=x)))
    o = np.array(pa["task_xgroup_off"]); o[1] = o[-1]
    cases.append((abi.KB_E_BADARG, dict(task_xgroup_off=o)))
    for code, ch in cases:
        with pytest.raises(engine.KbError) as ei:
            eng.load(_with(snap, **ch), PluginConf.default())
        assert ei.value.code == code, (ch.keys(), str(ei.value))


@pytest.mark.parametrize("labels,atoms", [(40, 1), (40, 0), (200, 0)])
def test_c3_host_spread_with_many_labels(eng, labels, atoms):
    """BASELINE config 3 with a tenth of the PodGroups under "one replica per host" over 40 / 200 labels (80 / 400 counter groups).
    80 groups fit the spare port-word bits (cycle_kernel, or the counter path with KB_AFF_ATOMS=0); 400 do not.  Engine vs the
    emulation."""
    s, conf = synth.make("c3")
    synth.add_host_spread(s, 0.1, labels=labels)
    e = util.emu_allocate(s, conf, mode=1)
    os.environ["KB_AFF_ATOMS"] = str(atoms)
    try:
        eng.load(s, conf)
    finally:
        os.environ.pop("KB_AFF_ATOMS", None)
    eng.allocate()
    r = eng.allocate()
    assert r.stats.pipeline == atoms
    util.assert_same_decisions(e.decisions, r.decisions, f"c3 + host spread over {labels} labels vs emulation")
    st = r.stats
    rec = {"workload": "c3", "groups": 2 * labels, "path": "cycle_kernel (groups as port-word atoms)" if atoms else "visit_kernel<0,1> (counters)",
           "spread_tasks": int(s.meta["spread_tasks"]), "gpu_ms": float(st.gpu_ms), "kernel_launches": int(st.kernel_launches),
           "allocated": int(st.tasks_allocated), "pairs_logical": int(st.pairs_logical), "pairs_per_s": float(st.pairs_logical) / (st.gpu_ms * 1e-3)}
    print("host spread timing:", json.dumps(rec))
