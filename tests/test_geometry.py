"""The launch-geometry sessions of tests/geometry_gen.py on the CPU: the node counts sit on the boundaries the restated geometry
names, the oracle reaches every deciding region, and the CPU emulation of the device algorithm (launch modes 0 / 1 / 5) agrees
with the oracle on them, so that a failure of tests/test_gpu_geometry.py points at the device, not at the shared logic."""
import numpy as np
import pytest

from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import geometry_gen as G
import util
from test_evict_parity import compare

H100 = G.Geometry(132)
CONF = PluginConf.default()


def test_boundaries_of_a_132_sm_h100():
    b = H100.boundaries()
    assert H100.tpi == 4 and H100.max_tpc == 12
    assert b["scan_pass2"] == b["evict_pass2"] == 67072 and b["scan_pass3"] == 134144
    assert b["prepass1_pass2"] == 8448 and b["prepass_pass2"] == 135168
    assert b["pipe_fallback"] == 201216 and b["pipe_tpc2"] == 16768
    assert G.Geometry(132, R=32).tpi == 1 and G.Geometry(132, R=32).boundaries()["scan_pass2"] == 16768
    assert G.Geometry(114).pipe_limit == 12 * 113 * 128          # H100 PCIe


@pytest.mark.parametrize("sm", [114, 132])
def test_node_counts_sit_on_the_boundaries(sm):
    geo = G.Geometry(sm)
    for name, b in geo.boundaries().items():
        below, at, above = G.boundary_ns(b)
        assert (below % 128, at % 128, above % 128) == (127, 0, 1), name
        if name.startswith("pipe_tpc"):
            k = int(name[len("pipe_tpc"):])
            assert geo.pipe_tpc(at) == k - 1 and geo.pipe_tpc(above) == k, name
        elif name == "pipe_fallback":
            assert geo.pipe_tpc(at) == geo.max_tpc and geo.pipe_tpc(above) == 0
        elif name.startswith("scan_pass"):
            p = int(name[-1])
            assert geo.scan_passes(at) == p - 1 and geo.scan_passes(above) == p, name
        elif name == "evict_pass2":
            assert geo.evict_passes(at) == 1 and geo.evict_passes(above) == 2
        elif name == "prepass1_pass2":
            assert geo.prepass1_passes(at) == 1 and geo.prepass1_passes(above) == 2
        elif name == "prepass_pass2":
            assert geo.prepass_passes(at) == 1 and geo.prepass_passes(above) == 2


def test_regions_sit_where_the_geometry_says(geo=H100):
    N = 201216
    r = G.regions(geo, N)
    assert all(geo.scan_pass_of(N, n) == geo.scan_passes(N) - 1 for n in r["late_scan"])
    assert all(geo.scan_pass_of(N, n) == 2 for n in r["scan_pass3"])
    assert all(geo.pipe_cta_of(N, n) == geo.pipe_S(N) - 1 for n in r["last_cta"])
    assert all(geo.evict_pass_of(N, n) >= 1 for n in r["evict_pass2"])
    assert [n // (geo.ag1(N) * 8) for n in r["prepass1_pass2"]] == [0, 1]
    assert [n // (geo.ag(N) * G.AFF_THREADS) for n in r["prepass_pass2"]] == [0, 1]
    for k in (31, 32, 33, 40):
        assert len(r[f"spread{k}"]) == k
    spread = [n for k in (31, 32, 33, 40) for n in r[f"spread{k}"]]
    assert len(set(spread)) == len(spread)


SMALL = [2000, 8449, 16769]


@pytest.mark.parametrize("N", SMALL)
def test_small_sessions_reach_their_regions_and_match_the_emulation(N):
    s = G.geometry_session(N, N, H100, background_jobs=2)
    o = kbo.allocate(s, CONF)
    cov = G.coverage(s, o, H100)
    assert cov["spread_full"] == [31, 32, 33, 40] and cov["alternations"] > 0, cov
    assert cov["gang_estar_chunks"] == [0, 1, 2, 3], cov
    assert all(v > 0 for v in cov["region_placements"].values()), cov
    for mode in (0, 1, 5):
        e = util.emu_allocate(s, CONF, mode=mode)
        util.assert_same_decisions(o.decisions, e.decisions, f"N={N} mode {mode}")
        ns, os_ = util.emu_states(e)
        util.assert_same_state(o, ns, os_, f"N={N} mode {mode}")


@pytest.mark.parametrize("kw", [{"pref": True}, {"pod_pref": True}], ids=["pref", "pod_pref"])
def test_affinity_sessions_match_the_emulation(kw):
    N = 8449
    s = G.geometry_session(N, 3, H100, background_jobs=2, **kw)
    o = kbo.allocate(s, CONF)
    assert G.coverage(s, o, H100)["spread_full"] == [31, 32, 33, 40]
    if kw.get("pod_pref"):
        assert G.far_node_placements(s, o)["prepass1_pass2"] == 3
    for mode in (0, 1, 5):
        e = util.emu_allocate(s, CONF, mode=mode)
        util.assert_same_decisions(o.decisions, e.decisions, f"{kw} mode {mode}")


def test_evict_session_matches_the_emulation():
    N = 3000
    s = G.geometry_session(N, 4, H100, evict=True, background_jobs=2)
    run = s.meta["running"]
    acts = ("reclaim", "allocate", "backfill", "preempt")
    o, ev, order = kbo.cycle(s, CONF, actions=acts, running=run)
    assert ev.sum() > 0
    for mode in (1, 5):
        g, gev, gorder = util.emu_cycle(s, CONF, acts, run, mode=mode)
        compare(f"evict mode {mode}", o, ev, order, g, gev, gorder, util.emu_states(g))


@pytest.mark.slow
@pytest.mark.parametrize("N", [H100.pipe_limit, H100.pipe_limit + 1])
def test_largest_sessions_match_the_emulation(N):
    s = G.geometry_session(N, 7, H100, background_jobs=2)
    o = kbo.allocate(s, CONF, threads=8)
    cov = G.coverage(s, o, H100)
    assert cov["max_scan_pass"] >= 2 and cov["last_tile_used"], cov
    e = util.emu_allocate(s, CONF, mode=1)
    util.assert_same_decisions(o.decisions, e.decisions, f"N={N}")
