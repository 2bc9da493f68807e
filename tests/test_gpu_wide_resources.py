"""Sessions with 9 to 32 resource dimensions through the C ABI (-m gpu): the sessions of test_wide_resources.py on the kernels'
wide instances, bit-exact against the oracle (decisions and dispatch steps, evictions in order, node / job / queue state,
kb_bind_list); kb_predicate_score / kb_best_nodes rows at R = 17; the C++ host mirror's cycle shells at R = 12; and a synthetic
cluster of ~5 000 tasks on 600 nodes (several node tiles per CTA, hundreds of evictions)."""
from __future__ import annotations

import numpy as np
import pytest

from kube_batch_b200 import engine, synth
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import aff_gen
import util
from test_evict_parity import compare, tier_variants
from test_gpu_many_queues import check_bind_list, check_cycle
from test_wide_resources import (ACTION_LISTS, CLUSTER_SEEDS, FULL_LIST, HAND_CASES, HAND_IDS, REFUSED_EVICT, affinity_session, evicted_high,
                                 random_cluster_builder, widen, widen_cluster)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("R", [9, 12, 17, 32])
def test_synthetic_sessions_on_the_gpu(R):
    eng = engine.Engine(0)
    for seed in range(2):
        s = synth.random_session(seed, tasks=300, jobs=40, nodes=40, queues=2, oversub=3.0, R=R)
        run = synth.running_of(s, 0.8, seed=seed + 1)
        for tname, conf in tier_variants():
            eng.load(s, conf).load_running(run)
            for acts in ACTION_LISTS:
                check_cycle(eng, s, conf, acts, run, f"R={R} seed {seed} {tname} {acts}")
            o = kbo.allocate(s, conf)
            r = eng.allocate()
            util.assert_same_decisions(o.decisions, r.decisions, f"R={R} {tname} kb_allocate")
            assert int(r.stats.pipeline) == 0
    eng.close()


@pytest.mark.parametrize("R", [9, 17, 32])
def test_object_clusters_with_running_pods_on_the_gpu(R):
    eng = engine.Engine(0)
    evictions = high = 0
    for seed in CLUSTER_SEEDS:
        s = widen_cluster(seed, R)
        for tname, conf in tier_variants():
            eng.load(s, conf).load_running(s.meta["running"])
            for acts in ACTION_LISTS:
                res, gev, gorder, bounds = eng.cycle(acts)
                o, ev, order = kbo.cycle(s, conf, actions=acts, running=s.meta["running"])
                compare(f"R={R} cluster {seed} {tname} {acts}", o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
                util.assert_same_decisions(o.decisions, res.decisions, f"R={R} cluster {seed} {tname} {acts}")
                check_bind_list(eng, o.decisions, f"R={R} cluster {seed} {tname} {acts}")
                evictions += int(gev.sum())
                high += evicted_high(s, gev)
    assert evictions > 0
    if R >= 17:
        assert high > 0, "no victim held a resource in dimension 8 or above"
    eng.close()


def run_on_gpu(s, tiers, acts=("allocate",), running=None):
    """kb_cycle of `acts` on a fresh engine against kbo.cycle: decisions, evictions in order, node / job / queue state, bind list"""
    running = running if running is not None else s.meta.get("running")
    o, ev, order = kbo.cycle(s, tiers, actions=acts, running=running)
    eng = engine.Engine(0).load(s, tiers).load_running(running)
    res, gev, gorder, _ = eng.cycle(acts)
    what = f"{acts}"
    compare(what, o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
    util.assert_same_decisions(o.decisions, res.decisions, what)
    check_bind_list(eng, o.decisions, what)
    eng.close()
    return o, ev


@pytest.mark.parametrize("case", HAND_CASES, ids=HAND_IDS)
def test_hand_computed_cases_on_the_gpu(case):
    case(run_on_gpu)


def test_affinity_sessions_at_12_dimensions_on_the_gpu():
    evicting = 0
    for seed in range(6):
        s = affinity_session(seed)
        for tname, conf in tier_variants():
            for acts in ACTION_LISTS:
                what = f"affinity {seed} {tname} {acts}"
                o, ev, order = kbo.cycle(s, conf, actions=acts, running=s.meta["running"])
                eng = engine.Engine(0).load(s, conf)                  # a fresh engine: no Running table left from an earlier load
                try:
                    eng.load_running(s.meta["running"])
                    loaded = True
                except engine.KbError as e:                          # refused for evicting actions; placing ones run without it
                    assert any(m in str(e) for m in REFUSED_EVICT), e
                    loaded = False
                try:
                    if not loaded and acts == FULL_LIST:
                        continue
                    try:
                        res, gev, gorder, _ = eng.cycle(acts)
                    except engine.KbError as e:
                        assert acts == FULL_LIST and any(m in str(e) for m in REFUSED_EVICT), e
                        continue
                    if not loaded:                                    # no Running table on the engine: nothing to evict either
                        assert not ev.any()
                        ev, order = ev[:0], order[:0]
                    evicting += acts == FULL_LIST
                    compare(what, o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
                    util.assert_same_decisions(o.decisions, res.decisions, what)
                    check_bind_list(eng, o.decisions, what)
                finally:
                    eng.close()
    assert evicting > 0


def test_predicate_score_and_best_nodes_at_17_dimensions():
    s = synth.random_session(5, tasks=200, jobs=30, nodes=300, R=17)
    conf = PluginConf.default()
    eng = engine.Engine(0).load(s, conf)
    fit, score = eng.predicate_score(0, s.T)
    for t in range(0, s.T, 7):                                        # kbo.predicate_score: one task per call
        rfit, rscore = kbo.predicate_score(s, conf, t)
        np.testing.assert_array_equal(fit[t], rfit, err_msg=f"task {t}: fit")
        np.testing.assert_array_equal(score[t][rfit != 0], rscore[rfit != 0], err_msg=f"task {t}: score")
    best = eng.best_nodes(0, s.T)
    key = np.where(fit != 0, (score + 0).astype(np.int64), -1)
    # best node: highest score among the feasible nodes, ties to the lowest index
    for t in range(s.T):
        if not fit[t].any():
            assert best[t] == 0
            continue
        n = int(np.argmax(key[t]))
        assert int(engine.key_node(np.array([best[t]]))[0]) == n, t
    assert fit.sum() > 0 and (~fit.astype(bool)).sum() > 0
    eng.close()


def test_cycle_shells_of_the_cpp_mirror_at_12_dimensions(tmp_path):
    import test_host_cpp_cycle as H
    H._build()
    b = widen(random_cluster_builder(11), 12, 11)
    assert b.flatten().R == 12
    cases = [(f"{tname}:{i}", acts, conf) for tname, conf in tier_variants() for i, acts in enumerate(ACTION_LISTS)]
    got = H.run_cases(tmp_path, b, cases)
    assert sorted(got) == sorted(label for label, _, _ in cases)
    for label, acts, conf in cases:
        H.compare_with_oracle(b, got[label], acts, conf, f"R=12 {label} {acts}")


def test_synthetic_cluster_with_hundreds_of_evictions_at_12_dimensions():
    s = synth.random_session(7, tasks=5000, jobs=500, nodes=600, queues=3, oversub=2.0, R=12)
    run = synth.running_of(s, 0.4)
    conf = PluginConf.default()
    eng = engine.Engine(0).load(s, conf).load_running(run)
    res, n = check_cycle(eng, s, conf, FULL_LIST, run, "R=12 synthetic 5000 tasks")
    assert n >= 100, n
    eng.close()


def test_the_shard_flag_on_one_rank_runs_wide_sessions():
    """KB_ENGINE_SHARD only matters with world > 1: one rank runs a wide session as usual"""
    from kube_batch_b200 import abi
    s = synth.random_session(9, tasks=60, jobs=8, nodes=20, R=9)
    eng = engine.Engine(0, flags=abi.KB_ENGINE_SHARD).load(s, PluginConf.default())
    util.assert_same_decisions(kbo.allocate(s, PluginConf.default()).decisions, eng.allocate().decisions, "R=9 one rank")
    eng.close()


def test_more_than_32_dimensions_are_refused_by_the_engine():
    from kube_batch_b200 import abi
    s = synth.random_session(1, tasks=40, jobs=6, nodes=8, R=32)
    cs, keep = s.to_c()
    cs.R = abi.KB_MAX_R + 1
    s.to_c = lambda: (cs, keep)
    eng = engine.Engine(0)
    with pytest.raises(engine.KbError) as ei:
        eng.load(s, PluginConf.default())
    assert ei.value.code == abi.KB_E_BADARG and "KB_MAX_R = 32" in str(ei.value)
    eng.close()
