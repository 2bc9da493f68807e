"""Sessions with more than 256 label, taint or host-port atoms through the C ABI (-m gpu): the sessions of test_many_atoms.py on
the kernels' wide-atom instances (W = 5..16), bit-exact against the oracle (decisions and dispatch steps, evictions in order,
node / job / queue state, kb_bind_list); kb_predicate_score / kb_best_nodes rows at W = 16; the hand-computed cases decided by
the atom at bit 1023; preferred node-affinity terms and host-level anti-affinity atoms past word 4; and the C++ host mirror's
flattener and cycle shells on the per-team cluster."""
from __future__ import annotations

import numpy as np
import pytest

from kube_batch_b200 import abi, engine, synth
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import util
from test_evict_parity import compare, tier_variants
from test_gpu_many_queues import check_bind_list, check_cycle
from test_many_atoms import (ACTION_LISTS, FULL_LIST, HAND, HI, TEAMS, _two_nodes, anti_affinity_cluster, anti_affinity_outcome, deepen, members_listed,
                             pref_decides, synthetic, team_cluster)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("pref", [False, True], ids=["required", "preferred"])
@pytest.mark.parametrize("W", [5, 8, 16])
def test_synthetic_sessions_on_the_gpu(W, pref):
    eng = engine.Engine(0)
    evictions = 0
    for seed in range(2):
        s = synthetic(W, seed, pref)
        if pref:                                                       # the preferred terms in the last word decide
            moved, evicted = pref_decides(s, synth.running_of(s, 0.8, seed=seed + 1))
            assert moved > 0 and evicted > 0, (moved, evicted)
        run = synth.running_of(s, 0.8, seed=seed + 1)
        for tname, conf in tier_variants():
            eng.load(s, conf).load_running(run)
            for acts in ACTION_LISTS:
                evictions += check_cycle(eng, s, conf, acts, run, f"W={W} seed {seed} {tname} {acts}")[1]
            o = kbo.allocate(s, conf)
            r = eng.allocate()
            util.assert_same_decisions(o.decisions, r.decisions, f"W={W} {tname} kb_allocate")
            assert int(r.stats.pipeline) == 0
    assert evictions > 0
    eng.close()


def _team(name: str) -> int:
    """team index of a pod or node name: ns/p123-0, ns/low123, n123"""
    base = name.split("/")[-1]
    return int("".join(ch for ch in base if ch.isdigit())[:3])


@pytest.mark.parametrize("selectors", ["label", "affinity"])
def test_per_team_cluster_on_the_gpu(selectors):
    s = team_cluster(selectors=selectors).flatten()
    assert s.W > 4
    conf = PluginConf.default()
    eng = engine.Engine(0).load(s, conf).load_running(s.meta["running"])
    for acts in (("allocate",), ("allocate", "backfill")):
        res, _ = check_cycle(eng, s, conf, acts, s.meta["running"], f"teams {selectors} {acts}")
    tasks, nodes = s.meta["tasks"], s.meta["nodes"]
    placed = [(t, int(n)) for t, n in enumerate(res.decisions["node"]) if n >= 0]
    assert len(placed) == TEAMS and all(_team(tasks[t]) == _team(nodes[n]) for t, n in placed)
    assert any(_team(nodes[n]) >= 256 for _, n in placed)            # placements decided by atoms in word 4
    eng.close()


def test_per_team_cluster_with_running_pods_on_the_gpu():
    s = team_cluster(running=True).flatten()
    run = s.meta["running"]
    eng = engine.Engine(0)
    evicted_hi = 0
    for tname, conf in tier_variants():
        eng.load(s, conf).load_running(run)
        res, gev, gorder, _ = eng.cycle(FULL_LIST)
        o, ev, order = kbo.cycle(s, conf, actions=FULL_LIST, running=run)
        what = f"teams running {tname}"
        compare(what, o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
        util.assert_same_decisions(o.decisions, res.decisions, what)
        check_bind_list(eng, o.decisions, what)
        evicted_hi += sum(1 for i in np.nonzero(gev)[0] if run["names"][i].split("/")[1].startswith("low") and _team(run["names"][i]) >= 256)
    assert evicted_hi > 0                                              # evictions on nodes whose taint atom sits in word 4
    eng.close()


def test_host_level_anti_affinity_past_word_4_on_the_gpu():
    import follow_oracle
    s = anti_affinity_cluster().flatten()
    assert s.W == 5 and s.pod_affinity is not None
    run = members_listed(s)
    eng = engine.Engine(0)
    for tname, conf in tier_variants():
        eng.load(s, conf).load_running(run)
        for acts in (("allocate",), FULL_LIST):
            o, ev, order = follow_oracle.cycle(s, conf, acts, run)
            res, gev, gorder, _ = eng.cycle(acts)
            what = f"anti-affinity {tname} {acts}"
            compare(what, o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
            util.assert_same_decisions(o.decisions, res.decisions, what)
            check_bind_list(eng, o.decisions, what)
            if tname == "default" and acts == FULL_LIST:
                assert anti_affinity_outcome(s, res.decisions, gev) == ("n03", ["ns/low-x"])
    # the groups became port atoms (bits 300 and 301), not counters: the matrix kernels take the session, which they refuse
    # for counter-path sessions
    eng.load(s, PluginConf.default())
    eng.best_nodes(0, s.T)
    eng.close()


@pytest.mark.parametrize("family", HAND)
def test_hand_computed_cases_on_the_gpu(family):
    s = _two_nodes(family)
    eng = engine.Engine(0).load(s, PluginConf.default())
    r = eng.allocate()
    assert int(r.decisions["node"][0]) == 1, r.decisions
    util.assert_same_decisions(kbo.allocate(s, PluginConf.default()).decisions, r.decisions, family)
    eng.close()


def test_predicate_score_and_best_nodes_at_16_words():
    s = deepen(synth.random_session(5, tasks=200, jobs=30, nodes=300, W=16), 5)
    conf = PluginConf.default()
    eng = engine.Engine(0).load(s, conf)
    fit, score = eng.predicate_score(0, s.T)
    for t in range(0, s.T, 7):                                        # kbo.predicate_score: one task per call
        rfit, rscore = kbo.predicate_score(s, conf, t)
        np.testing.assert_array_equal(fit[t], rfit, err_msg=f"task {t}: fit")
        np.testing.assert_array_equal(score[t][rfit != 0], rscore[rfit != 0], err_msg=f"task {t}: score")
    best = eng.best_nodes(0, s.T)
    key = np.where(fit != 0, (score + 0).astype(np.int64), -1)
    for t in range(s.T):
        if not fit[t].any():
            assert best[t] == 0
            continue
        assert int(engine.key_node(np.array([best[t]]))[0]) == int(np.argmax(key[t])), t
    sel = (s.task_sel_req[15] & HI) != 0                              # the selector atom at bit 1023 excludes nodes without it
    assert sel.any() and not fit[np.ix_(sel, (s.node_labels[15] & HI) == 0)].any()
    eng.close()


def test_cycle_shells_of_the_cpp_mirror_on_the_per_team_cluster(tmp_path):
    """kbhost.hpp's flattener and cycle shells (tests/host affinity_run) on the per-team cluster: every action list as one
    kb_cycle, allocate (+ backfill) also as per-action shells, against the oracle"""
    import test_host_cpp_affinity as HA
    HA._build()
    b = team_cluster(selectors="affinity", running=True)
    assert b.flatten().W > 4
    cases = [(f"{tname}:{i}:{mode}", acts, mode, conf) for tname, conf in tier_variants() for i, acts in enumerate(ACTION_LISTS)
             for mode in (("cycle",) if "reclaim" in acts else ("cycle", "shells"))]
    HA._check_cases(tmp_path, b, cases, "teams")


def test_refusals_by_the_engine():
    s = synth.random_session(1, tasks=40, jobs=6, nodes=8, W=16)
    cs, keep = s.to_c()
    cs.W = abi.KB_MAX_W + 1
    s.to_c = lambda: (cs, keep)
    eng = engine.Engine(0)
    with pytest.raises(engine.KbError) as ei:
        eng.load(s, PluginConf.default())
    assert ei.value.code == abi.KB_E_BADARG and "KB_MAX_W = 16" in str(ei.value)
    s = synth.random_session(1, tasks=40, jobs=6, nodes=8, R=9, W=5)
    with pytest.raises(engine.KbError) as ei:
        eng.load(s, PluginConf.default())
    assert ei.value.code == abi.KB_E_UNSUPPORTED_FEATURE and "KB_NARROW_R (8)" in str(ei.value) and "KB_NARROW_W (4)" in str(ei.value)
    eng.close()
