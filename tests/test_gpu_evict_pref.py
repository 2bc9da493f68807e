"""reclaim / preempt with preferred node affinity on the GPU (kb_evict_kernels.cu: pass 1 for the max count, then the sweep) through
the C ABI, against the oracle: the hand vectors, random clusters on both record geometries, host-level anti-affinity together with
the terms, and the synthetic cluster run twice from the loaded state."""
from __future__ import annotations

import numpy as np
import pytest

from kube_batch_b200 import abi, synth
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import util
from test_evict_parity import ACTION_LISTS, FULL_LIST, compare
from test_evict_pref import VECTORS, pref_cluster, pref_tiers, vector

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from kube_batch_b200 import engine
    e = engine.Engine(0)
    yield e
    e.close()


def _run(eng, acts):
    if len(acts) == 1:
        res, gev, gorder = eng.reclaim() if acts[0] == "reclaim" else eng.preempt()
        return res, gev, gorder
    res, gev, gorder, _ = eng.cycle(acts)
    return res, gev, gorder


def _check(eng, s, tiers, acts, what):
    o, ev, order = kbo.cycle(s, tiers, actions=acts, running=s.meta["running"])
    res, gev, gorder = _run(eng, acts)
    compare(what, o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
    util.assert_same_decisions(o.decisions, res.decisions, what)
    return res


@pytest.mark.parametrize("case", VECTORS, ids=lambda c: c[0].split(":")[0])
def test_hand_vectors_on_the_gpu(eng, case):
    name, kw, tiers, action, want, want_tainted = case
    for tainted in ((False, True) if want_tainted is not None else (False,)):
        s = vector(a_tainted=tainted, **kw)
        eng.load(s, tiers).load_running(s.meta["running"])
        res = _check(eng, s, tiers, (action,), f"{name} tainted={tainted}")
        assert [s.meta["nodes"][n] if n >= 0 else None for n in res.decisions["node"]] == (want_tainted if tainted else want), name


@pytest.mark.parametrize("seed", [1, 2, 3, 6, 7, 10, 13, 16])
def test_random_clusters_on_the_gpu(eng, seed):
    """odd seeds: the persistent pipeline's record geometry (R = 3, W = 2); even seeds: R = 2, W = 1 (per-visit kernels)"""
    s = pref_cluster(seed)
    if not (s.task_n_pref_terms > 0).any():
        pytest.skip("no pending pod with preferred terms drawn")
    for tname, tiers in pref_tiers():
        eng.load(s, tiers).load_running(s.meta["running"])
        for acts in (("reclaim",), ("preempt",)) + (ACTION_LISTS if seed % 3 == 1 else (FULL_LIST,)):
            _check(eng, s, tiers, acts, f"gpu seed {seed} {tname} {acts}")


@pytest.mark.parametrize("seed", range(2))
def test_larger_clusters_on_the_gpu(eng, seed):
    s = pref_cluster(100 + seed, big=True)
    for tname, tiers in pref_tiers():
        eng.load(s, tiers).load_running(s.meta["running"])
        for acts in (("preempt",), FULL_LIST):
            _check(eng, s, tiers, acts, f"gpu big seed {seed} {tname} {acts}")


@pytest.mark.parametrize("seed", [0, 1, 2, 11])
def test_host_level_anti_affinity_with_preferred_terms_on_the_gpu(eng, seed):
    s = pref_cluster(200 + seed, spread=True)
    if s.pod_affinity is None:
        pytest.skip("no spread group drawn")
    for tname, tiers in pref_tiers():
        eng.load(s, tiers).load_running(s.meta["running"])
        for acts in (("preempt",), FULL_LIST):
            _check(eng, s, tiers, acts, f"gpu spread seed {seed} {tname} {acts}")


def test_synthetic_cluster_with_preferred_terms_on_the_gpu(eng):
    s = synth.add_node_pref(synth.random_session(0, tasks=3000, jobs=300, nodes=600, queues=3, oversub=2.0), 0.3)
    run = synth.running_of(s, 0.4)
    o, ev, order = kbo.cycle(s, PluginConf.default(), actions=FULL_LIST, running=run)
    assert int(ev.sum()) > 500
    eng.load(s, PluginConf.default()).load_running(run)
    for rep in range(2):                                                    # repeatable from the loaded state
        res, gev, gorder, bounds = eng.cycle(FULL_LIST)
        compare(f"gpu synthetic rep {rep}", o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
        util.assert_same_decisions(o.decisions, res.decisions, f"gpu synthetic rep {rep}")
        assert int(res.stats.evictions) == int(ev.sum())
