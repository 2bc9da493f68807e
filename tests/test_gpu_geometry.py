"""`-m gpu`: sessions whose deciding nodes sit where the launch geometry splits the node table (tests/geometry_gen.py), from
the first to the last tile count cycle_kernel takes and beyond, through the C ABI against the oracle, bit for bit: decisions and
dispatch steps, evictions in order, node / job / queue state and kb_bind_list.  The node counts come from the restated geometry
of THIS device's SM count.  The oracle runs once per session and conf; its result is reused across engine modes.  Each test prints
the geometry it reached (-s)."""
import os

import numpy as np
import pytest

from kube_batch_b200 import abi, engine, synth
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import geometry_gen as G
import util
from test_evict_parity import compare
from test_gpu_many_queues import check_bind_list

pytestmark = pytest.mark.gpu

CONF = PluginConf.default()
CYCLE = ("reclaim", "allocate", "backfill", "preempt")
THREADS = os.cpu_count() or 1


@pytest.fixture(scope="module")
def geo():
    return G.Geometry(G.device_sm())


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(device=0)
    yield e
    e.close()


def _oracle(s, conf=CONF, actions=kbo.KBO_ACTION_ALLOCATE):
    return kbo.allocate(s, conf, threads=THREADS, actions=actions)


def _check(eng, s, o, what, conf=CONF, backfill=False):
    eng.load(s, conf)
    r = eng.allocate()
    if backfill:
        r = eng.backfill()
    util.assert_same_decisions(o.decisions, r.decisions, what)
    util.assert_same_state(o, eng.node_state(), eng.order_state(), what)
    st = r.stats
    assert (st.tasks_processed, st.tasks_allocated, st.tasks_pipelined, st.visits, st.jobs_ready) == \
        (o.result.tasks_processed, o.result.tasks_allocated, o.result.tasks_pipelined, o.result.visits, o.result.jobs_ready), what
    check_bind_list(eng, o.decisions, what)
    return r


def _assert_reached(cov, geo, N, what):
    """The deciding regions of the session were all used by the oracle."""
    reg = G.regions(geo, N)
    rp = cov["region_placements"]
    for name in ("last", "late_scan", "scan_pass3", "last_cta", "prepass1_pass2", "prepass_pass2"):
        if name in reg:
            assert rp.get(name, 0) > 0, (what, name, cov)
    assert cov["spread_full"] == [31, 32, 33, 40], (what, cov)
    assert cov["alternations"] > 0 and cov["last_tile_used"], (what, cov)
    assert cov["gang_estar_chunks"] == [0, 1, 2, 3], (what, cov)


def _pipe_ns(geo):
    """One N per tile count 1..max_tpc: the first N of the count (N % 128 == 1), its last N (== 0) or one below (== 127)."""
    s1 = geo.sm - 1
    out = []
    for k in range(1, geo.max_tpc + 1):
        lo, hi = (k - 1) * s1 * G.TILE + 1, k * s1 * G.TILE
        out.append([lo, hi - 1, hi][k % 3])
    return out


def test_pipeline_at_every_tile_count_per_scanner_cta(eng, geo):
    seen = []
    for k, N in enumerate(_pipe_ns(geo), start=1):
        s = G.geometry_session(N, 10 + k, geo, background_jobs=2)
        o = _oracle(s)
        cov = G.coverage(s, o, geo)
        _assert_reached(cov, geo, N, f"tpc {k}")
        r = _check(eng, s, o, f"pipeline N={N}")
        assert r.stats.pipeline == 1 and geo.pipe_tpc(N) == k, (N, k)
        seen.append(k)
        print(f"\npipeline N={N}: {geo.describe(N)}, last CTA used {cov['last_cta_used']}")
    assert seen == list(range(1, 13)) if geo.max_tpc == 12 else seen


@pytest.fixture(scope="module")
def at_fallback(geo):
    """The last N on cycle_kernel and the first one past it, with their oracle results."""
    out = {}
    for N in (geo.pipe_limit, geo.pipe_limit + 1):
        s = G.geometry_session(N, 7, geo, background_jobs=2)
        out[N] = (s, _oracle(s))
    return out


def test_pipeline_fallback_boundary(eng, geo, at_fallback):
    for N, (s, o) in at_fallback.items():
        cov = G.coverage(s, o, geo)
        _assert_reached(cov, geo, N, f"N={N}")
        r = _check(eng, s, o, f"fallback N={N}")
        want = 1 if N <= geo.pipe_limit else 0
        print(f"\nN={N}: stats.pipeline {r.stats.pipeline}, {geo.describe(N)}")
        assert r.stats.pipeline == want, (N, r.stats.pipeline)


@pytest.mark.parametrize("flags", [abi.KB_ENGINE_NO_PIPE, abi.KB_ENGINE_NO_PIPE | abi.KB_ENGINE_FORCE_OVERLAP,
                                   abi.KB_ENGINE_NO_PIPE | abi.KB_ENGINE_CHAIN2, abi.KB_ENGINE_NO_PIPE | abi.KB_ENGINE_CHAIN4],
                         ids=["no_pipe", "force_overlap", "chain2", "chain4"])
def test_per_visit_modes_at_three_scan_passes(geo, at_fallback, flags):
    e = engine.Engine(device=0, flags=flags)
    try:
        if flags & (abi.KB_ENGINE_CHAIN2 | abi.KB_ENGINE_CHAIN4):
            # kb_session_load lowers the chain length from the record width alone (R = 3 / W = 2 here, as in c2): the chain kernel
            # serves look-ahead visits on c2 with this engine, so the sessions below run it too (whether they hit is their own)
            c2, c2conf = synth.make("c2")
            e.load(c2, c2conf)
            assert e.allocate().stats.chain_hits > 0, flags
        for N, (s, o) in at_fallback.items():
            assert geo.scan_passes(N) >= 3
            r = _check(e, s, o, f"flags {flags} N={N}")
            assert r.stats.pipeline == 0
            if flags & abi.KB_ENGINE_FORCE_OVERLAP:        # the scanners ran ahead with the replayer's exclusions
                assert r.stats.predictions > 0, (flags, N)
            print(f"\nflags {flags:#x} N={N}: scan passes {geo.scan_passes(N)}, grid {geo.scan_grid(N)}, "
                  f"chain hits {r.stats.chain_hits}, overlap predictions {r.stats.predictions}")
    finally:
        e.close()


@pytest.mark.parametrize("R", [4, 32])
def test_per_visit_wide_records_at_two_scan_passes(eng, R):
    geo = G.Geometry(G.device_sm(), R=R)
    N = geo.boundaries()["scan_pass2"] + 1
    s = G.geometry_session(N, 20 + R, geo, background_jobs=2)
    o = _oracle(s)
    _assert_reached(G.coverage(s, o, geo), geo, N, f"R={R}")
    r = _check(eng, s, o, f"R={R} N={N}")
    assert r.stats.pipeline == 0 and geo.scan_passes(N) == 2
    print(f"\nR={R} N={N}: {geo.describe(N)}")


def test_backfill_after_allocate_at_three_scan_passes(eng, geo):
    N = geo.boundaries()["scan_pass3"] + 1
    s = G.geometry_session(N, 31, geo, background_jobs=2)
    o = _oracle(s, actions=kbo.KBO_ACTION_ALLOCATE | kbo.KBO_ACTION_BACKFILL)
    cov = G.coverage(s, o, geo)
    _assert_reached(cov, geo, N, f"backfill N={N}")
    assert cov["backfill_slots_past_estar_chunk"] > 0, cov
    _check(eng, s, o, f"backfill N={N}", backfill=True)
    print(f"\nbackfill N={N}: {geo.describe(N)}, PodGroups whose backfill slots cross into a chunk past e*'s: "
          f"{cov['backfill_slots_past_estar_chunk']}")


def test_shipped_action_list_with_victims_in_the_second_sweep_pass(eng, geo):
    N = geo.boundaries()["evict_pass2"] + 513
    s = G.geometry_session(N, 41, geo, evict=True, background_jobs=2)
    run = s.meta["running"]
    o, ev, order = kbo.cycle(s, CONF, actions=CYCLE, running=run, threads=THREADS)
    cov = G.coverage(s, o, geo, ev)
    assert geo.evict_passes(N) == 2 and cov["evictions"] > 0 and cov["max_evict_pass_of_victim"] == 1, cov
    eng.load(s, CONF).load_running(run)
    res, gev, gorder, _ = eng.cycle(CYCLE)
    compare(f"cycle N={N}", o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
    util.assert_same_decisions(o.decisions, res.decisions, f"cycle N={N}")
    check_bind_list(eng, o.decisions, f"cycle N={N}")
    print(f"\ncycle N={N}: {geo.describe(N)}, evictions {cov['evictions']} (victim pass {cov['max_evict_pass_of_victim']})")


@pytest.mark.parametrize("which", ["prepass1_pass2", "prepass_pass2"])
def test_counter_path_past_the_prepass_grids(eng, geo, which):
    N = geo.boundaries()[which] + 1
    s = G.geometry_session(N, 51, geo, pod_pref=True, background_jobs=2)
    o = _oracle(s)
    cov = G.coverage(s, o, geo)
    _assert_reached(cov, geo, N, which)
    far = G.far_node_placements(s, o)
    assert far.get(which, 0) > 0, (which, far)
    _check(eng, s, o, f"counter path N={N}")
    print(f"\ncounter path N={N}: {geo.describe(N)}, placements on the far node of each prepass region {far}")


def test_preferred_node_affinity_max_count_only_in_the_last_cta(eng, geo, at_fallback):
    for N in at_fallback:
        s = G.geometry_session(N, 61, geo, pref=True, background_jobs=2)
        o = _oracle(s)
        far = s.meta["pref_region"]
        assert G.coverage(s, o, geo)["region_placements"][far] > 0
        r = _check(eng, s, o, f"pref N={N}")
        print(f"\npreferred node affinity N={N}: pipeline {r.stats.pipeline}, max-count nodes in {far}")


def test_predicate_score_and_best_nodes_at_the_largest_n(eng, geo, at_fallback):
    N = max(at_fallback)
    s, _ = at_fallback[N]
    eng.load(s, CONF)
    rows = [0, s.T // 3, s.T - 1] + [int(s.job_task_off[j]) for j in s.meta["class_region"]][:4]
    for t in rows:
        fit, score = eng.predicate_score(t, t + 1)
        of, osc = kbo.predicate_score(s, CONF, t)
        np.testing.assert_array_equal(of, fit[0], err_msg=f"fit row {t}")
        np.testing.assert_array_equal(osc, score[0], err_msg=f"score row {t}")
        best = int(engine.key_node(eng.best_nodes(t, t + 1))[0])
        exp = int(np.argmax(np.where(of > 0, osc, -np.inf))) if of.any() else -1
        assert best == exp, (t, best, exp)
    print(f"\npredicate / score rows {rows} at N={N}")
